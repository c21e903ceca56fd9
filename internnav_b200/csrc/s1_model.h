// System-1 (NavDP) executor: RGB-D encoder, goal compressor, noise predictor and the DDPM sampling loop, as host-side
// C++ that sequences the kernels in this directory.  Mirrors NavDP_Policy_DPT_CriticSum_DAT (reference
// internnav/model/basemodel/internvla_n1/navdp.py L16-312) and DAT_RGBD_Patch_Backbone / TokenCompressor
// (internnav/model/encoder/navdp_backbone.py L60-202).
#pragma once
#include <vector>

#include "n1_ops.h"
#include "s1_kernels.h"
#include "weights.h"

namespace n1 {

struct Lin {
  bf16* w = nullptr;  // [N, ldw] bf16, K-major
  float* b = nullptr;  // [N] fp32 or null
  int N = 0, K = 0, ldw = 0;
};
// out[M, N] = A[M, K] @ L.w^T with L's bias (if any) in the epilogue
inline void linear(const Lin& L, const bf16* A, int lda, void* out, int ldo, int M, GemmEpilogue e, cudaStream_t s) {
  e.bias = L.b;
  gemm_bf16(A, lda, L.w, L.ldw, out, ldo, M, L.N, L.K, e, s);
}
struct LNp {
  float* w = nullptr;
  float* b = nullptr;
};

// Caller-provided scratch, carved with a bump pointer.  With base == nullptr it only measures.
class Carver {
 public:
  Carver(void* base, size_t bytes) : base_(static_cast<char*>(base)), cap_(bytes) {}
  template <typename T>
  T* take(size_t n) {
    const size_t bytes = (n * sizeof(T) + 255) & ~size_t(255);
    char* p = base_ ? base_ + off_ : nullptr;
    off_ += bytes;
    if (base_ && off_ > cap_) throw Error(-7, "workspace too small: need > " + std::to_string(off_) + " bytes");
    return reinterpret_cast<T*>(p);
  }
  size_t used() const { return off_; }
  bool dry() const { return base_ == nullptr; }

 private:
  char* base_;
  size_t cap_, off_ = 0;
};

struct S1Dims {
  int D = 384;          // token_dim
  int heads = 8;        // decoder / former heads (hd 48)
  int layers = 16;      // temporal_depth
  int T = 32;           // predict_size (out_pos_embed rows)
  int frames = 2;       // memory_size
  int vlm_dim = 3584;   // latent width
  int n_query = 4;      // latent tokens per env
  int ddpm_steps = 20;  // num_train_timesteps
  // Stand-alone NavDP policy (NavDPNet, internnav/model/basemodel/navdp/navdp_policy.py): RGBDBackbone sees `frames` RGB
  // frames but ONE depth frame, the condition row is [time, goal, goal, goal, memory tokens], there is no VLM goal path,
  // and a critic head ranks the sampled trajectories.  Defaults = the InternVLA-N1 head.
  int frames_depth = 0;  // 0: as many depth frames as RGB frames
  int goal_slots = 1;    // condition tokens that carry the goal embedding
  int standalone = 0;    // 1: NavDPNet wiring (no vlm_embed_mlp / goal_compressor, fp32 ImageNet constants, critic head)
  int depth_frames() const { return frames_depth > 0 ? frames_depth : frames; }
  int mem_tokens() const { return 16 * frames; }
  int cond_tokens() const { return 1 + goal_slots + mem_tokens(); }
};

class S1Model {
 public:
  S1Dims dims;
  void load(const WeightSource& ws, const S1Dims& d, cudaStream_t s);
  bool loaded() const { return loaded_; }

  // rgb fp32 [B, frames, 224, 224, 3] in [0,1]; depth fp32 [B, frames, 224, 224(,1)] metres -> out bf16 [B, 16*frames, D]
  size_t ws_rgbd(int B) const;
  void rgbd_encode(void* ws, size_t ws_bytes, const float* rgb, const float* depth, bf16* out, int B,
                   cudaStream_t s) const;
  // Training branch (s1_train.cu): the tokens of the FROZEN RGB ViT for the
  // [goal frame, current frame] pairs, as the Q-former sees them -- final LayerNorm, cls dropped, former_pe added --
  // mem bf16 [B, 2 * frames * 256, D]: only the first frames * 256 rows of every environment are written.
  size_t ws_rgb_tokens(int B) const;
  void rgb_tokens(void* ws, size_t ws_bytes, const float* rgb, bf16* mem, int B, cudaStream_t s) const;
  // latents bf16 [B, n_query, vlm_dim] -> goal bf16 [B, 1, D]
  size_t ws_goal(int B) const;
  void goal_compress(void* ws, size_t ws_bytes, const bf16* latents, bf16* goal, int B, cudaStream_t s) const;
  // One noise prediction.  x_t fp32 [B*Ns, T, 3]; timesteps int32 [B] (device) or null -> t_scalar for all;
  // goal [B,1,D], rgbd [B,16*frames,D] bf16 -> eps fp32 [B*Ns, T, 3]
  size_t ws_denoise(int B, int Ns, int T) const;
  void navdp_eps(void* ws, size_t ws_bytes, const float* x_t, const int* tsteps, int t_scalar, const bf16* goal,
                 const bf16* rgbd, float* eps, int B, int Ns, int T, cudaStream_t s) const;
  // Whole K-step ancestral sampling loop.  x_init fp32 [B*Ns,T,3]; step_noise fp32 [K-1, B*Ns, T, 3] (noise for
  // t = K-1 .. 1 in that order); traj_out fp32 [B*Ns, T, 3].
  void navdp_sample(void* ws, size_t ws_bytes, const bf16* goal, const bf16* rgbd, const float* x_init,
                    const float* step_noise, float* traj_out, int B, int Ns, int T, int K, cudaStream_t s) const;

  // Critic of the stand-alone policy (navdp_policy.py L172-187 `predict_critic`): trajectories fp32 [B*Ns, T, 3], memory
  // tokens bf16 [B, mem_tokens, D] -> critic fp32 [B*Ns].  Full self-attention, cross-attention restricted to the memory
  // tokens (the time / goal slots are masked: `cond_critic_mask`), LayerNorm, mean over T, critic_head.
  void navdp_critic(void* ws, size_t ws_bytes, const float* traj, const bf16* rgbd, float* critic, int B, int Ns, int T,
                    cudaStream_t s) const;

  static void ddpm_tables(int N, std::vector<DdpmCoef>& coef);

 private:
  struct VitBlock {
    LNp n1, n2;
    Lin qkv, proj, fc1, fc2;
    float *ls1 = nullptr, *ls2 = nullptr;
  };
  struct Vit {
    Lin patch;
    float* pos_patch = nullptr;  // [256, D] fp32, bicubic-resampled
    float* cls_pos = nullptr;    // [D] cls + pos[0]
    std::vector<VitBlock> blk;
    LNp norm;
  };
  struct DecLayer {
    LNp n1, n2, n3;
    Lin sa_qkv, sa_out, ca_q, ca_kv, ca_out, ff1, ff2;
  };
  struct DenoiseBufs;

  Vit load_vit(const WeightSource& ws, bool depth, cudaStream_t s);
  DecLayer load_dec_layer(const WeightSource& ws, bool with_kv, cudaStream_t s);
  size_t vit_forward(const Vit& v, Carver c, const float* img, bool depth, int n_img, bf16* mem, int slot_base,
                     cudaStream_t s, bool with_pe = true, int frames_per_env = 0) const;
  size_t rgbd_impl(Carver c, const float* rgb, const float* depth, bf16* out, int B, cudaStream_t s) const;
  size_t goal_impl(Carver c, const bf16* latents, bf16* goal, int B, cudaStream_t s) const;
  DenoiseBufs carve_denoise(Carver& c, int B, int Ns, int T) const;
  bool fused_attn(int T) const;
  void decoder_pass(const DenoiseBufs& d, const float* x_t, const int* tsteps, int t_scalar, bool cond_full,
                    const bf16* goal, const bf16* rgbd, int B, int Ns, int T, int mode, float* x_io,
                    const float* noise, float* eps, const DdpmCoef& cf, cudaStream_t s) const;

  Arena arena_;
  bool loaded_ = false;
  Vit rgb_, depth_;
  float* former_pe_ = nullptr;     // [frames*2*256, D]
  bf16* former_query_ = nullptr;   // [16*frames, D]
  std::vector<DecLayer> former_;
  Lin project_;
  // goal path
  Lin vlm0_, vlm1_, vlm2_;
  float* token_pe_ = nullptr;      // [n_query, D]
  bf16* goal_q_ = nullptr;         // [1, D] projected constant query
  Lin goal_kv_, goal_out_;
  // denoiser
  float *in_w_ = nullptr, *in_b_ = nullptr;  // input_embed [D,3], [D]
  float* out_pos_ = nullptr;                 // [T, D]
  float* cond_pos_ = nullptr;                // [2+16*frames, D]
  std::vector<DecLayer> dec_;
  Lin kv_all_;                               // all layers' cross-attention K/V projections stacked: [layers*2D, D]
  LNp final_ln_;
  float *head_w_ = nullptr, *head_b_ = nullptr;
  float *critic_w_ = nullptr, *critic_b_ = nullptr;  // stand-alone policy only: critic_head [1, D], [1]
};

}  // namespace n1
