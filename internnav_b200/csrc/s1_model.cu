// System-1 (NavDP) executor.  See s1_model.h for the reference mapping.
#include "s1_model.h"

#include <math.h>

#include <vector>

namespace n1 {

namespace {

Lin load_lin(Arena& a, const WeightSource& ws, const std::string& wname, const std::string& bname, long row0, long rows,
             long cols, cudaStream_t s) {
  Lin L;
  L.N = (int)rows;
  L.K = (int)((cols + 7) & ~7L);
  L.w = ws.mat(a, wname, row0, rows, cols, &L.ldw, s);
  if (!bname.empty()) L.b = ws.f32_rows(a, bname, row0, rows, 1, s);
  N1_CHECK(L.N % 8 == 0, "linear " + wname + ": N must be a multiple of 8");
  return L;
}
LNp load_ln(Arena& a, const WeightSource& ws, const std::string& prefix, cudaStream_t s) {
  LNp p;
  p.w = ws.f32(a, prefix + ".weight", s);
  p.b = ws.f32(a, prefix + ".bias", s);
  return p;
}

// torch.nn.functional.interpolate(mode="bicubic", scale_factor=s, antialias=False, align_corners=False) restated
// for the DINOv2 position table (dinov2.py L180-211): [G*G, D] -> [g*g, D] with the *given* scale factor
// (src = (dst + 0.5) / s - 0.5, A = -0.75, border-clamped taps), fp32 like ATen's upsample_bicubic2d.
void bicubic_resample(const std::vector<float>& src, int G, int g, int D, float scale_factor, std::vector<float>& dst) {
  dst.assign((size_t)g * g * D, 0.f);
  const float rscale = (float)(1.0 / (double)scale_factor);
  const float A = -0.75f;
  auto cc1 = [&](float x) { return ((A + 2.f) * x - (A + 3.f)) * x * x + 1.f; };
  auto cc2 = [&](float x) { return ((A * x - 5.f * A) * x + 8.f * A) * x - 4.f * A; };
  auto coeffs = [&](float t, float* c) {
    c[0] = cc2(t + 1.f), c[1] = cc1(t), c[2] = cc1(1.f - t), c[3] = cc2(2.f - t);
  };
  auto clampi = [&](int v) { return v < 0 ? 0 : (v > G - 1 ? G - 1 : v); };
  for (int oy = 0; oy < g; ++oy) {
    const float sy = rscale * (oy + 0.5f) - 0.5f;
    const int iy = (int)floorf(sy);
    float cy[4];
    coeffs(sy - iy, cy);
    for (int ox = 0; ox < g; ++ox) {
      const float sx = rscale * (ox + 0.5f) - 0.5f;
      const int ix = (int)floorf(sx);
      float cx[4];
      coeffs(sx - ix, cx);
      float* o = &dst[((size_t)oy * g + ox) * D];
      for (int i = 0; i < 4; ++i) {
        const int yy = clampi(iy - 1 + i);
        for (int j = 0; j < 4; ++j) {
          const int xx = clampi(ix - 1 + j);
          const float w = cy[i] * cx[j];
          const float* sp = &src[((size_t)yy * G + xx) * D];
          for (int d = 0; d < D; ++d) o[d] += w * sp[d];
        }
      }
    }
  }
}

}  // namespace

// ------------------------------------------------------------------------------------------------ load
S1Model::Vit S1Model::load_vit(const WeightSource& ws, bool depth, cudaStream_t s) {
  const int D = dims.D;
  Vit v;
  // patch embed: Conv2d weight [D, 3, 14, 14] -> GEMM weight [D, 588]; depth folds the 3 identical channels.
  if (!depth) {
    v.patch = load_lin(arena_, ws, "patch_embed.proj.weight", "patch_embed.proj.bias", 0, D, 588, s);
  } else {
    const SrcTensor& w = ws.get("patch_embed.proj.weight");
    float* folded = arena_.alloc_n<float>((size_t)D * 196);
    fold_groups(w.data, w.dtype, D, 3, 196, folded, s);
    v.patch.N = D, v.patch.K = 200, v.patch.ldw = 200;
    v.patch.w = arena_.alloc_n<bf16>((size_t)D * 200);
    pack2d(folded, 0, 196, 0, D, 196, v.patch.w, 1, 200, s);
    v.patch.b = ws.f32(arena_, "patch_embed.proj.bias", s);
  }
  // position table: bicubic 37x37 -> 16x16 once (input is always 224x224), cls handled separately
  {
    const SrcTensor& pe = ws.get("pos_embed");
    const long ntok = pe.numel() / D;
    const int G = (int)lround(sqrt((double)(ntok - 1)));
    N1_CHECK((long)G * G + 1 == ntok, "pos_embed is not 1 + G*G tokens");
    float* dev = ws.f32(arena_, "pos_embed", s);
    float* cls = ws.f32(arena_, "cls_token", s);
    std::vector<float> host((size_t)ntok * D), hcls(D);
    N1_CUDA(cudaStreamSynchronize(s));
    N1_CUDA(cudaMemcpy(host.data(), dev, host.size() * 4, cudaMemcpyDeviceToHost));
    N1_CUDA(cudaMemcpy(hcls.data(), cls, D * 4, cudaMemcpyDeviceToHost));
    std::vector<float> grid(host.begin() + D, host.end()), out;
    if (G == 16) {
      out = grid;
    } else {
      const float sf = (float)((16 + 0.1) / (double)G);  // interpolate_offset = 0.1 (dinov2.py L196-199)
      bicubic_resample(grid, G, 16, D, sf, out);
    }
    v.pos_patch = arena_.alloc_n<float>(256 * D);
    N1_CUDA(cudaMemcpy(v.pos_patch, out.data(), out.size() * 4, cudaMemcpyHostToDevice));
    for (int d = 0; d < D; ++d) hcls[d] += host[d];
    v.cls_pos = arena_.alloc_n<float>(D);
    N1_CUDA(cudaMemcpy(v.cls_pos, hcls.data(), D * 4, cudaMemcpyHostToDevice));
  }
  v.blk.resize(12);
  for (int i = 0; i < 12; ++i) {
    const WeightSource b = ws.sub("blocks." + std::to_string(i) + ".");
    VitBlock& k = v.blk[i];
    k.n1 = load_ln(arena_, b, "norm1", s);
    k.n2 = load_ln(arena_, b, "norm2", s);
    k.qkv = load_lin(arena_, b, "attn.qkv.weight", "attn.qkv.bias", 0, 3 * D, D, s);
    k.proj = load_lin(arena_, b, "attn.proj.weight", "attn.proj.bias", 0, D, D, s);
    k.fc1 = load_lin(arena_, b, "mlp.fc1.weight", "mlp.fc1.bias", 0, 4 * D, D, s);
    k.fc2 = load_lin(arena_, b, "mlp.fc2.weight", "mlp.fc2.bias", 0, D, 4 * D, s);
    k.ls1 = b.f32(arena_, "ls1.gamma", s);
    k.ls2 = b.f32(arena_, "ls2.gamma", s);
  }
  v.norm = load_ln(arena_, ws, "norm", s);
  return v;
}

S1Model::DecLayer S1Model::load_dec_layer(const WeightSource& ws, bool with_kv, cudaStream_t s) {
  const int D = dims.D;
  DecLayer L;
  L.n1 = load_ln(arena_, ws, "norm1", s);
  L.n2 = load_ln(arena_, ws, "norm2", s);
  L.n3 = load_ln(arena_, ws, "norm3", s);
  L.sa_qkv = load_lin(arena_, ws, "self_attn.in_proj_weight", "self_attn.in_proj_bias", 0, 3 * D, D, s);
  L.sa_out = load_lin(arena_, ws, "self_attn.out_proj.weight", "self_attn.out_proj.bias", 0, D, D, s);
  L.ca_q = load_lin(arena_, ws, "multihead_attn.in_proj_weight", "multihead_attn.in_proj_bias", 0, D, D, s);
  if (with_kv)
    L.ca_kv = load_lin(arena_, ws, "multihead_attn.in_proj_weight", "multihead_attn.in_proj_bias", D, 2 * D, D, s);
  L.ca_out = load_lin(arena_, ws, "multihead_attn.out_proj.weight", "multihead_attn.out_proj.bias", 0, D, D, s);
  const long ff = ws.get("linear1.bias").numel();
  L.ff1 = load_lin(arena_, ws, "linear1.weight", "linear1.bias", 0, ff, D, s);
  L.ff2 = load_lin(arena_, ws, "linear2.weight", "linear2.bias", 0, D, ff, s);
  return L;
}

void S1Model::load(const WeightSource& ws, const S1Dims& d, cudaStream_t s) {
  dims = d;
  const int D = dims.D;
  N1_CHECK(D == 384, "System-1 kernels are specialised for token_dim 384");
  N1_CHECK(D / dims.heads == 48, "System-1 decoder head_dim must be 48");
  const int Mq = dims.mem_tokens();
  const long slots = dims.frames + dims.depth_frames();   // 256-token image slots of the Q-former memory
  rgb_ = load_vit(ws.sub("rgbd_encoder.rgb_model."), false, s);
  depth_ = load_vit(ws.sub("rgbd_encoder.depth_model."), true, s);
  const WeightSource enc = ws.sub("rgbd_encoder.");
  {
    const long pe_rows = enc.get("former_pe.weight").numel() / D;
    N1_CHECK(pe_rows >= slots * 256, "former_pe too small (needs navdp_version > 0 layout)");
    former_pe_ = enc.f32_rows(arena_, "former_pe.weight", 0, slots * 256, D, s);
    int ld;
    former_query_ = enc.mat(arena_, "former_query.weight", 0, Mq, D, &ld, s);
  }
  former_.clear();
  for (int i = 0; i < 2; ++i)
    former_.push_back(load_dec_layer(enc.sub("former_net.layers." + std::to_string(i) + "."), true, s));
  project_ = load_lin(arena_, enc, "project_layer.weight", "project_layer.bias", 0, D, D, s);

  // goal path: vlm_embed_mlp (navdp.py L94-100) + TokenCompressor (navdp_backbone.py L60-99); the stand-alone policy has
  // none (its goal token is point_encoder(goal) or zero, computed by the caller)
  if (!dims.standalone) {
  vlm0_ = load_lin(arena_, ws, "vlm_embed_mlp.0.weight", "vlm_embed_mlp.0.bias", 0, dims.vlm_dim / 4, dims.vlm_dim, s);
  vlm1_ = load_lin(arena_, ws, "vlm_embed_mlp.2.weight", "vlm_embed_mlp.2.bias", 0, dims.vlm_dim / 8, dims.vlm_dim / 4, s);
  vlm2_ = load_lin(arena_, ws, "vlm_embed_mlp.4.weight", "vlm_embed_mlp.4.bias", 0, D, dims.vlm_dim / 8, s);
  const WeightSource gc = ws.sub("goal_compressor.");
  token_pe_ = gc.f32_rows(arena_, "token_positional_encoding.position_embedding.weight", 0, dims.n_query, D, s);
  goal_kv_ = load_lin(arena_, gc, "cross_attention.in_proj_weight", "cross_attention.in_proj_bias", D, 2 * D, D, s);
  goal_out_ = load_lin(arena_, gc, "cross_attention.out_proj.weight", "cross_attention.out_proj.bias", 0, D, D, s);
  {
    // constant query: (target_embedding[0] + query_pe[0]) @ Wq^T + bq, computed once
    Lin gq = load_lin(arena_, gc, "cross_attention.in_proj_weight", "cross_attention.in_proj_bias", 0, D, D, s);
    float* te = gc.f32_rows(arena_, "target_embedding.weight", 0, 1, D, s);
    float* qp = gc.f32_rows(arena_, "query_positional_encoding.position_embedding.weight", 0, 1, D, s);
    std::vector<float> a(D), b(D);
    N1_CUDA(cudaStreamSynchronize(s));
    N1_CUDA(cudaMemcpy(a.data(), te, D * 4, cudaMemcpyDeviceToHost));
    N1_CUDA(cudaMemcpy(b.data(), qp, D * 4, cudaMemcpyDeviceToHost));
    for (int i = 0; i < D; ++i) a[i] += b[i];
    N1_CUDA(cudaMemcpy(te, a.data(), D * 4, cudaMemcpyHostToDevice));
    bf16* qin = arena_.alloc_n<bf16>(8 * D);
    N1_CUDA(cudaMemsetAsync(qin, 0, 8 * D * sizeof(bf16), s));
    f32_to_bf16(te, qin, D, s);
    goal_q_ = arena_.alloc_n<bf16>(D);
    linear(gq, qin, D, goal_q_, D, 1, GemmEpilogue(), s);
  }
  }  // !standalone

  // denoiser
  in_w_ = ws.f32(arena_, "input_embed.weight", s);
  in_b_ = ws.f32(arena_, "input_embed.bias", s);
  out_pos_ = ws.f32_rows(arena_, "out_pos_embed", 0, dims.T, D, s);
  cond_pos_ = ws.f32_rows(arena_, "cond_pos_embed", 0, dims.cond_tokens(), D, s);
  if (dims.standalone) {
    critic_w_ = ws.f32(arena_, "critic_head.weight", s);
    critic_b_ = ws.f32(arena_, "critic_head.bias", s);
  }
  dec_.clear();
  kv_all_.N = dims.layers * 2 * D, kv_all_.K = D, kv_all_.ldw = D;
  kv_all_.w = arena_.alloc_n<bf16>((size_t)kv_all_.N * D);
  kv_all_.b = arena_.alloc_n<float>(kv_all_.N);
  for (int i = 0; i < dims.layers; ++i) {
    const WeightSource lw = ws.sub("decoder.layers." + std::to_string(i) + ".");
    dec_.push_back(load_dec_layer(lw, false, s));
    const SrcTensor& w = lw.get("multihead_attn.in_proj_weight");
    const SrcTensor& b = lw.get("multihead_attn.in_proj_bias");
    pack2d(w.data, w.dtype, D, D, 2 * D, D, kv_all_.w + (size_t)i * 2 * D * D, 1, D, s);
    pack2d(b.data, b.dtype, 1, D, 2 * D, 1, kv_all_.b + (size_t)i * 2 * D, 0, 1, s);
  }
  final_ln_ = load_ln(arena_, ws, "layernorm", s);
  head_w_ = ws.f32(arena_, "action_head.weight", s);
  head_b_ = ws.f32(arena_, "action_head.bias", s);
  N1_CUDA(cudaStreamSynchronize(s));
  loaded_ = true;
}

// ------------------------------------------------------------------------------------------------ RGB-D encoder
// Returns the scratch high-water mark (bytes from the start of `c0`'s buffer); launches nothing when dry.
size_t S1Model::vit_forward(const Vit& v, Carver c, const float* img, bool depth, int n_img, bf16* mem, int slot_base,
                            cudaStream_t s, bool with_pe, int frames_per_env) const {
  if (frames_per_env <= 0) frames_per_env = dims.frames;
  const int D = dims.D;
  const long rows = (long)n_img * 257;
  const int ldk = v.patch.K;
  bf16* col = c.take<bf16>((size_t)n_img * 256 * ldk);
  bf16* x = c.take<bf16>(rows * D);
  bf16* ln = c.take<bf16>(rows * D);
  bf16* qkv = c.take<bf16>(rows * 3 * D);
  bf16* att = c.take<bf16>(rows * D);
  bf16* hid = c.take<bf16>(rows * 4 * D);
  if (c.dry()) return c.used();

  if (depth)
    patchify_depth(img, col, n_img, ldk, s);
  else
    patchify_rgb(img, col, n_img, ldk, s, dims.standalone != 0);
  {
    GemmEpilogue e;  // x[img, 1 + p, :] = patch + bias + pos[p]
    e.rows_per_group = 256, e.group_stride = 257, e.group_offset = 1, e.row_add = v.pos_patch;
    linear(v.patch, col, ldk, x, D, n_img * 256, e, s);
  }
  fill_cls(x, v.cls_pos, n_img, 257, D, s);
  for (const VitBlock& b : v.blk) {
    layernorm(x, D, ln, D, b.n1.w, b.n1.b, (int)rows, D, 1e-6f, 0, s);
    linear(b.qkv, ln, D, qkv, 3 * D, (int)rows, GemmEpilogue(), s);
    AttnParams p = {};
    p.q = qkv, p.k = qkv + D, p.v = qkv + 2 * D, p.o = att;
    p.ldq = p.ldk = p.ldv = 3 * D, p.ldo = D;
    p.heads_q = p.heads_kv = 6, p.hd = 64, p.batch = n_img, p.seq_q = p.seq_k = 257, p.kv_div = 1;
    p.scale = 0.125f;
    attention(p, s);
    GemmEpilogue e1;
    e1.gamma = b.ls1, e1.residual = x, e1.ldr = D;
    linear(b.proj, att, D, x, D, (int)rows, e1, s);
    layernorm(x, D, ln, D, b.n2.w, b.n2.b, (int)rows, D, 1e-6f, 0, s);
    GemmEpilogue e2;
    e2.act = ACT_GELU;
    linear(b.fc1, ln, D, hid, 4 * D, (int)rows, e2, s);
    GemmEpilogue e3;
    e3.gamma = b.ls2, e3.residual = x, e3.ldr = D;
    linear(b.fc2, hid, 4 * D, x, D, (int)rows, e3, s);
  }
  vit_out(x, mem, v.norm.w, v.norm.b, with_pe ? former_pe_ : nullptr, n_img, frames_per_env, slot_base,
          dims.frames + dims.depth_frames(), s);
  return c.used();
}

size_t S1Model::rgbd_impl(Carver c, const float* rgb, const float* depth, bf16* out, int B, cudaStream_t s) const {
  const int D = dims.D, F = dims.frames, Fd = dims.depth_frames(), Mq = dims.mem_tokens();
  const long mrows = (long)B * (F + Fd) * 256;
  bf16* mem = c.take<bf16>(mrows * D);
  const long qrows = (long)B * Mq;
  bf16* x = c.take<bf16>(qrows * D);
  bf16* y = c.take<bf16>(qrows * D);
  bf16* qkv = c.take<bf16>(qrows * 3 * D);
  bf16* att = c.take<bf16>(qrows * D);
  bf16* hid = c.take<bf16>(qrows * 2048);
  bf16* kv = c.take<bf16>(mrows * 2 * D);
  // the two ViT passes run back to back on one stream and share the scratch after `kv`
  const size_t hi_rgb = vit_forward(rgb_, c, rgb, false, B * F, mem, 0, s);
  const size_t hi_dep = vit_forward(depth_, c, depth, true, B * Fd, mem, F, s, true, Fd);
  const size_t hi = hi_rgb > hi_dep ? hi_rgb : hi_dep;
  if (c.dry()) return hi;

  // Q-former: 2 post-norm decoder layers, queries = former_query (navdp_backbone.py L194-201)
  bcast_rows(former_query_, x, qrows, Mq, D, s);
  const float scale48 = 1.0f / sqrtf(48.f);
  for (const DecLayer& L : former_) {
    linear(L.sa_qkv, x, D, qkv, 3 * D, (int)qrows, GemmEpilogue(), s);
    AttnParams p = {};
    p.q = qkv, p.k = qkv + D, p.v = qkv + 2 * D, p.o = att;
    p.ldq = p.ldk = p.ldv = 3 * D, p.ldo = D;
    p.heads_q = p.heads_kv = dims.heads, p.hd = 48, p.batch = B, p.seq_q = p.seq_k = Mq, p.kv_div = 1;
    p.scale = scale48;
    attention(p, s);
    GemmEpilogue e;
    e.residual = x, e.ldr = D;
    linear(L.sa_out, att, D, y, D, (int)qrows, e, s);
    layernorm(y, D, x, D, L.n1.w, L.n1.b, (int)qrows, D, 1e-5f, 0, s);

    linear(L.ca_q, x, D, qkv, D, (int)qrows, GemmEpilogue(), s);
    linear(L.ca_kv, mem, D, kv, 2 * D, (int)mrows, GemmEpilogue(), s);
    AttnParams pc = {};
    pc.q = qkv, pc.k = kv, pc.v = kv + D, pc.o = att;
    pc.ldq = D, pc.ldk = pc.ldv = 2 * D, pc.ldo = D;
    pc.heads_q = pc.heads_kv = dims.heads, pc.hd = 48, pc.batch = B, pc.seq_q = Mq, pc.seq_k = (F + Fd) * 256;
    pc.kv_div = 1, pc.scale = scale48;
    attention(pc, s);
    linear(L.ca_out, att, D, y, D, (int)qrows, e, s);
    layernorm(y, D, x, D, L.n2.w, L.n2.b, (int)qrows, D, 1e-5f, 0, s);

    GemmEpilogue er;
    er.act = ACT_RELU;
    linear(L.ff1, x, D, hid, L.ff1.N, (int)qrows, er, s);
    linear(L.ff2, hid, L.ff1.N, y, D, (int)qrows, e, s);
    layernorm(y, D, x, D, L.n3.w, L.n3.b, (int)qrows, D, 1e-5f, 0, s);
  }
  linear(project_, x, D, out, D, (int)qrows, GemmEpilogue(), s);
  return hi;
}

size_t S1Model::ws_rgbd(int B) const { return rgbd_impl(Carver(nullptr, 0), nullptr, nullptr, nullptr, B, nullptr); }
void S1Model::rgbd_encode(void* ws, size_t ws_bytes, const float* rgb, const float* depth, bf16* out, int B,
                          cudaStream_t s) const {
  N1_CHECK(loaded_, "System-1 weights not loaded");
  N1_CHECK(ws != nullptr, "null workspace");
  if (ws_bytes < ws_rgbd(B)) throw Error(-7, "rgbd_encode: workspace too small");
  rgbd_impl(Carver(ws, ws_bytes), rgb, depth, out, B, s);
}

// ------------------------------------------------------------------------------------------------ goal token
size_t S1Model::goal_impl(Carver c, const bf16* latents, bf16* goal, int B, cudaStream_t s) const {
  const int D = dims.D, nq = dims.n_query;
  const long rows = (long)B * nq;
  bf16* h1 = c.take<bf16>(rows * vlm0_.N);
  bf16* h2 = c.take<bf16>(rows * vlm1_.N);
  bf16* tok = c.take<bf16>(rows * D);
  bf16* kv = c.take<bf16>(rows * 2 * D);
  bf16* q = c.take<bf16>((long)B * D);
  bf16* att = c.take<bf16>((long)B * D);
  if (c.dry()) return c.used();
  GemmEpilogue relu;
  relu.act = ACT_RELU;
  linear(vlm0_, latents, dims.vlm_dim, h1, vlm0_.N, (int)rows, relu, s);
  linear(vlm1_, h1, vlm0_.N, h2, vlm1_.N, (int)rows, relu, s);
  GemmEpilogue pe;  // + token positional encoding (row % n_query)
  pe.rows_per_group = nq, pe.group_stride = nq, pe.group_offset = 0, pe.row_add = token_pe_;
  linear(vlm2_, h2, vlm1_.N, tok, D, (int)rows, pe, s);
  linear(goal_kv_, tok, D, kv, 2 * D, (int)rows, GemmEpilogue(), s);
  bcast_rows(goal_q_, q, B, 1, D, s);
  AttnParams p = {};
  p.q = q, p.k = kv, p.v = kv + D, p.o = att;
  p.ldq = D, p.ldk = p.ldv = 2 * D, p.ldo = D;
  p.heads_q = p.heads_kv = dims.heads, p.hd = 48, p.batch = B, p.seq_q = 1, p.seq_k = nq, p.kv_div = 1;
  p.scale = 1.0f / sqrtf(48.f);
  attention(p, s);
  linear(goal_out_, att, D, goal, D, B, GemmEpilogue(), s);
  return c.used();
}
size_t S1Model::ws_goal(int B) const { return goal_impl(Carver(nullptr, 0), nullptr, nullptr, B, nullptr); }
void S1Model::goal_compress(void* ws, size_t ws_bytes, const bf16* latents, bf16* goal, int B, cudaStream_t s) const {
  N1_CHECK(loaded_, "System-1 weights not loaded");
  N1_CHECK(ws != nullptr, "null workspace");
  if (ws_bytes < ws_goal(B)) throw Error(-7, "goal_compress: workspace too small");
  goal_impl(Carver(ws, ws_bytes), latents, goal, B, s);
}

// ------------------------------------------------------------------------------------------------ denoiser
struct S1Model::DenoiseBufs {
  bf16 *x, *x2, *ln, *qkv, *att, *hid, *cond, *ckv;
  int* klen;  // [B] visible memory-token count per environment (critic pass)
};

// Whether a sampling / eps pass over horizon T runs each decoder layer as the three fused kernels (self-attention block,
// cross-attention block, FF block) instead of the 9-launch sequence.  The blocks cover D = 384 / 8 heads (load() checks
// both), T <= 32, <= 64 condition tokens and contiguous weights; the critic pass (mode 2) always takes the sequence.
bool S1Model::fused_attn(int T) const {
  const int D = dims.D;
  if (!loaded_ || T > 32 || dims.cond_tokens() > 64) return false;
  for (const DecLayer& L : dec_)
    if (L.sa_qkv.ldw != D || L.sa_out.ldw != D || L.ca_q.ldw != D || L.ca_out.ldw != D || L.ff1.N != 1536 ||
        L.ff1.ldw != D || L.ff2.ldw != 1536)
      return false;
  return true;
}

S1Model::DenoiseBufs S1Model::carve_denoise(Carver& c, int B, int Ns, int T) const {
  const int D = dims.D, Mtok = dims.cond_tokens();
  const long R = (long)B * Ns * T;
  DenoiseBufs d = {};
  d.x = c.take<bf16>(R * D);
  d.x2 = c.take<bf16>(R * D);  // ping-pong partner of x for the fused GEMM + LayerNorm (no in-place update there)
  if (!fused_attn(T) || dims.standalone) {  // the 9-launch layer can run (the stand-alone policy's critic pass takes it)
    d.ln = c.take<bf16>(R * D);
    d.qkv = c.take<bf16>(R * 3 * D);
    d.att = c.take<bf16>(R * D);
  }
  d.hid = c.take<bf16>(R * 4 * D);
  d.cond = c.take<bf16>((long)B * Mtok * D);
  d.ckv = c.take<bf16>((long)B * Mtok * kv_all_.N);
  d.klen = c.take<int>(B);
  return d;
}

// One pass of the 16-layer decoder over all B*Ns*T rows (navdp.py L177-195).  `cond_slots`: 0 = condition tokens and
// their K/V are already in the workspace except the time token (slot 0), 1 = rebuild everything.
void S1Model::decoder_pass(const DenoiseBufs& d, const float* x_t, const int* tsteps, int t_scalar, bool cond_full,
                           const bf16* goal, const bf16* rgbd, int B, int Ns, int T, int mode, float* x_io,
                           const float* noise, float* eps, const DdpmCoef& cf, cudaStream_t s) const {
  const int D = dims.D, Mtok = dims.cond_tokens();
  const long R = (long)B * Ns * T;
  const int ldkv = kv_all_.N;
  const bool critic = mode == 2;  // stand-alone policy's predict_critic: no causal mask, memory tokens only, critic head
  const int kv_first = critic ? 1 + dims.goal_slots : 0, kv_len = Mtok - kv_first;
  embed_actions(x_t, in_w_, in_b_, out_pos_, d.x, R, T, s);
  if (cond_full) {
    build_cond(tsteps, t_scalar, goal, rgbd, cond_pos_, d.cond, B, Mtok, 0, Mtok, s, dims.goal_slots);
    linear(kv_all_, d.cond, D, d.ckv, ldkv, B * Mtok, GemmEpilogue(), s);
  } else {
    // only the time token changed: refresh row 0 of every environment (strided A and out)
    build_cond(tsteps, t_scalar, goal, rgbd, cond_pos_, d.cond, B, Mtok, 0, 1, s, dims.goal_slots);
    linear(kv_all_, d.cond, Mtok * D, d.ckv, Mtok * ldkv, B, GemmEpilogue(), s);
  }
  bf16* xc = d.x;   // current residual stream
  if (!critic && fused_attn(T)) {
    for (int l = 0; l < dims.layers; ++l) {
      const DecLayer& L = dec_[l];
      dec_sa_block(xc, D, L.n1.w, L.n1.b, 1e-5f, L.sa_qkv.w, L.sa_qkv.b, L.sa_out.w, L.sa_out.b, B, Ns, T, 1, s);
      dec_ca_block(xc, D, L.n2.w, L.n2.b, 1e-5f, L.ca_q.w, L.ca_q.b, L.ca_out.w, L.ca_out.b, d.ckv + (long)l * 2 * D, ldkv,
                   Mtok, B, Ns, T, s);
      ff_block_384(xc, D, L.n3.w, L.n3.b, 1e-5f, L.ff1.w, L.ff1.b, L.ff2.w, L.ff2.b, xc, D, (int)R, s);
    }
    head_ddpm(xc, final_ln_.w, final_ln_.b, head_w_, head_b_, R, mode, x_io, noise, eps, cf, s);
    return;
  }
  const float scale48 = 1.0f / sqrtf(48.f);
  // residual GEMM (N = 384) and the LayerNorm that follows it
  auto res_gemm_ln = [&](const Lin& W, const bf16* A, int lda, const LNp* ln) {
    GemmEpilogue res;
    res.residual = xc, res.ldr = D;
    linear(W, A, lda, xc, D, (int)R, res, s);
    if (ln) layernorm(xc, D, d.ln, D, ln->w, ln->b, (int)R, D, 1e-5f, 0, s);
  };
  layernorm(xc, D, d.ln, D, dec_[0].n1.w, dec_[0].n1.b, (int)R, D, 1e-5f, 0, s);
  for (int l = 0; l < dims.layers; ++l) {
    const DecLayer& L = dec_[l];
    linear(L.sa_qkv, d.ln, D, d.qkv, 3 * D, (int)R, GemmEpilogue(), s);
    AttnParams p = {};
    p.q = d.qkv, p.k = d.qkv + D, p.v = d.qkv + 2 * D, p.o = d.att;
    p.ldq = p.ldk = p.ldv = 3 * D, p.ldo = D;
    p.heads_q = p.heads_kv = dims.heads, p.hd = 48, p.batch = B * Ns, p.seq_q = p.seq_k = T, p.kv_div = 1;
    p.causal = critic ? 0 : 1, p.scale = scale48;
    attention(p, s);
    res_gemm_ln(L.sa_out, d.att, D, &L.n2);

    linear(L.ca_q, d.ln, D, d.qkv, D, (int)R, GemmEpilogue(), s);
    AttnParams pc = {};
    pc.q = d.qkv, pc.k = d.ckv + (long)l * 2 * D, pc.v = d.ckv + (long)l * 2 * D + D, pc.o = d.att;
    pc.ldq = D, pc.ldk = pc.ldv = ldkv, pc.ldo = D;
    pc.heads_q = pc.heads_kv = dims.heads, pc.hd = 48, pc.batch = B * Ns, pc.seq_q = T, pc.seq_k = Mtok;
    pc.kv_div = Ns, pc.scale = scale48;
    if (kv_first > 0) {
      // `cond_critic_mask` (navdp_policy.py L131-132): the time / goal slots are invisible -> every environment's keys are
      // the kv_len memory tokens; var-len addressing skips the masked rows without copying
      pc.k += (long)kv_first * ldkv, pc.v += (long)kv_first * ldkv;
      pc.k_len = d.klen, pc.k_slot = Mtok, pc.seq_k = kv_len;   // slotted addressing: env e owns rows [e * Mtok, +kv_len)
    }
    attention(pc, s);
    const bool ffb = L.ff1.N == 1536 && L.ff1.ldw == D && L.ff2.ldw == 1536;  // the weights fit the FF-block kernel
    res_gemm_ln(L.ca_out, d.att, D, ffb ? nullptr : &L.n3);  // the FF-block kernel applies norm3 itself

    const LNp* next_ln = l + 1 < dims.layers ? &dec_[l + 1].n1 : nullptr;  // the head applies the final LayerNorm itself
    if (ffb) {
      ff_block_384(xc, D, L.n3.w, L.n3.b, 1e-5f, L.ff1.w, L.ff1.b, L.ff2.w, L.ff2.b, xc, D, (int)R, s);
      if (next_ln) layernorm(xc, D, d.ln, D, next_ln->w, next_ln->b, (int)R, D, 1e-5f, 0, s);
    } else {
      GemmEpilogue gelu;
      gelu.act = ACT_GELU;
      linear(L.ff1, d.ln, D, d.hid, 4 * D, (int)R, gelu, s);
      res_gemm_ln(L.ff2, d.hid, 4 * D, next_ln);
    }
  }
  if (critic) {
    critic_head(xc, final_ln_.w, final_ln_.b, critic_w_, critic_b_, (long)B * Ns, T, eps, s);
    return;
  }
  head_ddpm(xc, final_ln_.w, final_ln_.b, head_w_, head_b_, R, mode, x_io, noise, eps, cf, s);
}

size_t S1Model::ws_denoise(int B, int Ns, int T) const {
  Carver c(nullptr, 0);
  carve_denoise(c, B, Ns, T);
  return c.used();
}

void S1Model::navdp_eps(void* ws, size_t ws_bytes, const float* x_t, const int* tsteps, int t_scalar, const bf16* goal,
                        const bf16* rgbd, float* eps, int B, int Ns, int T, cudaStream_t s) const {
  N1_CHECK(loaded_, "System-1 weights not loaded");
  N1_CHECK(ws != nullptr, "null workspace");
  N1_CHECK(T >= 1 && T <= dims.T, "predict horizon exceeds out_pos_embed");
  Carver c(ws, ws_bytes);
  DenoiseBufs d = carve_denoise(c, B, Ns, T);
  decoder_pass(d, x_t, tsteps, t_scalar, true, goal, rgbd, B, Ns, T, 0, nullptr, nullptr, eps, DdpmCoef(), s);
}

void S1Model::navdp_critic(void* ws, size_t ws_bytes, const float* traj, const bf16* rgbd, float* critic, int B, int Ns, int T,
                           cudaStream_t s) const {
  N1_CHECK(loaded_ && dims.standalone && critic_w_, "navdp_critic: needs the stand-alone NavDP policy weights");
  N1_CHECK(ws != nullptr && traj && rgbd && critic, "navdp_critic: null buffers");
  N1_CHECK(T >= 1 && T <= dims.T, "predict horizon exceeds out_pos_embed");
  Carver c(ws, ws_bytes);
  DenoiseBufs d = carve_denoise(c, B, Ns, T);
  fill_int(d.klen, dims.mem_tokens(), B, s);
  // nogoal embedding = zeros in every time / goal slot (navdp_policy.py L174-181); those slots are masked anyway
  decoder_pass(d, traj, nullptr, 0, true, nullptr, rgbd, B, Ns, T, 2, nullptr, nullptr, critic, DdpmCoef(), s);
}

// diffusers 0.33.1 DDPMScheduler(num_train_timesteps=N, beta_schedule="squaredcos_cap_v2", clip_sample=True,
// prediction_type="epsilon", variance_type="fixed_small"), set_timesteps(N): see SURVEY.md App. B / oracle/ddpm.py.
void S1Model::ddpm_tables(int N, std::vector<DdpmCoef>& coef) {
  auto abar = [](double u) {
    const double c = cos((u + 0.008) / 1.008 * M_PI / 2.0);
    return c * c;
  };
  std::vector<float> acp(N);
  float prod = 1.f;
  for (int i = 0; i < N; ++i) {
    double beta = 1.0 - abar((double)(i + 1) / N) / abar((double)i / N);
    if (beta > 0.999) beta = 0.999;
    const float alpha = 1.0f - (float)beta;
    prod *= alpha;
    acp[i] = prod;
  }
  coef.resize(N);
  for (int t = 0; t < N; ++t) {
    const float a_t = acp[t], a_prev = t > 0 ? acp[t - 1] : 1.0f;
    const float beta_prod_t = 1.f - a_t, beta_prod_prev = 1.f - a_prev;
    const float cur_alpha = a_t / a_prev, cur_beta = 1.f - cur_alpha;
    DdpmCoef c;
    c.sqrt_one_minus_acp = sqrtf(beta_prod_t);
    c.inv_sqrt_acp = 1.0f / sqrtf(a_t);
    c.c0 = sqrtf(a_prev) * cur_beta / beta_prod_t;
    c.c1 = sqrtf(cur_alpha) * beta_prod_prev / beta_prod_t;
    float var = beta_prod_prev / beta_prod_t * cur_beta;
    if (var < 1e-20f) var = 1e-20f;
    c.sigma = t > 0 ? sqrtf(var) : 0.f;
    coef[t] = c;
  }
}

void S1Model::navdp_sample(void* ws, size_t ws_bytes, const bf16* goal, const bf16* rgbd, const float* x_init,
                           const float* step_noise, float* traj_out, int B, int Ns, int T, int K,
                           cudaStream_t s) const {
  N1_CHECK(loaded_, "System-1 weights not loaded");
  N1_CHECK(ws != nullptr, "null workspace");
  N1_CHECK(T >= 1 && T <= dims.T, "predict horizon exceeds out_pos_embed");
  N1_CHECK(K >= 1, "need at least one denoising step");
  Carver c(ws, ws_bytes);
  DenoiseBufs d = carve_denoise(c, B, Ns, T);
  std::vector<DdpmCoef> coef;
  ddpm_tables(K, coef);
  const long n = (long)B * Ns * T * 3;
  if (traj_out != x_init) N1_CUDA(cudaMemcpyAsync(traj_out, x_init, n * sizeof(float), cudaMemcpyDeviceToDevice, s));
  for (int i = 0; i < K; ++i) {
    const int t = K - 1 - i;  // set_timesteps(K) with K == num_train_timesteps: t = K-1 .. 0 (navdp.py L247-250)
    const float* noise = (t > 0 && step_noise) ? step_noise + (long)i * n : nullptr;
    decoder_pass(d, traj_out, nullptr, t, i == 0, goal, rgbd, B, Ns, T, 1, traj_out, noise, nullptr, coef[t], s);
  }
}

}  // namespace n1
