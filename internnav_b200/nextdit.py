"""NextDiT System 1 (`system1 = "nextdit_async"`, the released DualVLN trajectory head, and the synchronous
`system1 = "nextdit"` head) on libn1b200.so.

Mirrors the nextdit branch of `InternVLAN1ForCausalLM.generate_traj` (internnav/model/basemodel/internvla_n1/
internvla_n1.py L349-432) for a batch of environments:

    latents [B, 4, 3584] + frames [B, 2, 224, 224, 3]
      -> condition tokens [B, 36, 768]     cond_projector | DINOv2 ViT-S -> MemoryEncoder -> QFormer   (arch L76-145)
      -> 10 flow-matching Euler steps of the 12-block LuminaNextDiT (nextdit_traj.py L125-178, L296-368) over
         B * Ns trajectories of 32 steps, classifier-free guidance batch [null | cond]
      -> trajectories [B * Ns, 32, 3]

The synchronous head (`asynchronous=False`) has no RGB branch (no rgb_model / memory_encoder / rgb_resampler,
internvla_n1_arch.py L131-145): its condition tokens are cond_projector(latents) alone, [B, n_query, 768] (internvla_n1.py
L361-382), and the frames are accepted and ignored, as in the reference.  The sampler is the same code with 4 keys per
cross-attention instead of 36.

Every matrix product, attention, normalisation and the sampler update run in the library (wgmma GEMM, the attention
kernels, csrc/nextdit_kernels.cu); this module is the schedule -- it orders the launches, owns the packed weights and the
per-call conditioning tables.  PyTorch is used for buffers and for a handful of per-CALL shape operations on tensors of a
few kilobytes (concatenating the condition tokens, the 10 x groups modulation inputs); nothing per trajectory row.

What is hoisted out of the denoising loop (the reference recomputes it every step; the values are step-independent):
  * the caption projection, the cross-attention K / V of all 12 blocks (keys depend only on the condition tokens),
  * the timestep embeddings of all 10 steps and from them ALL modulation vectors (12 blocks x 4 x 384 per group) in one GEMM.
Folded at load time: norm1_context's weight into to_k / to_v, tanh(gate) into to_v, norm_out.linear_2 into action_decoder,
the ImageNet normalisation into the patch embedding.
With guidance_scale == 1 the guided prediction `u + 1 * (c - u)` equals the conditional one up to one bf16 rounding, and the
null half of the batch is skipped unless `exact_cfg=True`.

The CUDA extension is mandatory: there is no CPU path (importing this module without a CUDA device works, calling it fails).
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from . import _bwd, _lib
from ._lib import ACT_GELU, ACT_GELU_TANH, ACT_NONE, ACT_RELU, ACT_SILU, ACT_SWIGLU, MOD_GATED_RESIDUAL, MOD_LN_SCALE, MOD_RMS_SCALE

DIM, HEADS, HD, LAYERS, LATENT, FFN = 384, 6, 64, 12, 768, 1024
RESNET_MEAN = (0.485, 0.456, 0.406)
RESNET_STD = (0.229, 0.224, 0.225)


def _resample_pos_embed(pos_embed, side=16, offset=0.1):
    """DinoVisionTransformer.interpolate_pos_encoding (dinov2.py L180-211) for a 224 x 224 input: bicubic resampling of the
    37 x 37 table, scale-factor form with interpolate_offset 0.1.  Done once at load time."""
    pe = pos_embed.float()
    n = pe.shape[1] - 1
    src = int(math.isqrt(n))
    if src == side:
        return pe
    s = float(side + offset) / src
    patch = F.interpolate(pe[:, 1:].reshape(1, src, src, -1).permute(0, 3, 1, 2), scale_factor=(s, s), mode="bicubic",
                          antialias=False)
    assert patch.shape[-1] == side and patch.shape[-2] == side
    return torch.cat((pe[:, :1], patch.permute(0, 2, 3, 1).reshape(1, side * side, -1)), dim=1)


def flow_match_schedule(n, num_train_timesteps=1000):
    """FlowMatchEulerDiscreteScheduler().set_timesteps(n, sigmas=np.linspace(1, 1 / n, n)) (internvla_n1.py L395-396; shift
    1.0, no dynamic shifting): -> (int64 timesteps [n] as the DiT receives them, float32 sigmas [n + 1] with the trailing 0)."""
    sig = torch.from_numpy(np.linspace(1.0, 1 / n, n).astype(np.float32)).to(torch.float32)
    return (sig * num_train_timesteps).to(torch.long), torch.cat((sig, torch.zeros(1)))


def fold_patch_embed(Wp, bp):
    """Conv2d(3, 384, 14, stride 14) on (x - mean) / std  ==  im2col(x) @ W'^T + b' with the ImageNet statistics folded in:
    W' [384, 3 x 200] (196 taps + 4 zero columns per channel, the layout of n1_op_patchify_depth), b' [384]; fp32."""
    Wp, bp = Wp.float(), bp.float()
    cols, bias = [], bp.clone()
    for c in range(3):
        wc = Wp[:, c].reshape(Wp.shape[0], 196)
        cols.append(F.pad(wc / RESNET_STD[c], (0, 4)))
        bias -= (RESNET_MEAN[c] / RESNET_STD[c]) * wc.sum(1)
    return torch.cat(cols, dim=1), bias.contiguous()


def fold_cross_kv(to_k, to_v, ctx_weight, gate, head_dim=64):
    """Cross-attention of LuminaNextDiTBlock (nextdit_traj.py L149-160) with the constants folded into the projections:
    K = to_k(RMSNorm(enc) * ctx) = RMSNorm_noweight(enc) @ (to_k * ctx)^T and, because the gate multiplies the attention
    OUTPUT per head (softmax(..) V_h * tanh(gate_h)), V' = to_v * ctx with its rows of head h scaled by tanh(gate_h)."""
    ctx = ctx_weight.float()
    g = torch.tanh(gate.float()).repeat_interleave(head_dim)
    return to_k.float() * ctx[None, :], to_v.float() * ctx[None, :] * g[:, None]


def fold_head(W2, b2, Wd, bd):
    """action_decoder(norm_out.linear_2(y)) as one [3 -> 8 rows, 384] product (rows 3..7 zero: GEMM N % 8 == 0)."""
    W2, b2, Wd, bd = W2.float(), b2.float(), Wd.float(), bd.float()
    return F.pad(Wd @ W2, (0, 0, 0, 5)), F.pad(Wd @ b2 + bd, (0, 5)).contiguous()


class NextDiTSystem1:
    """state_dict keys: internnav_b200.manifest.nextdit_shapes(asynchronous=...) (the reference's attribute paths below
    `.model`).  asynchronous=True: `system1 = "nextdit_async"`; False: `system1 = "nextdit"`."""
    asynchronous = True

    def __init__(self, device="cuda:0", num_inference_steps=10, asynchronous=True):
        self.device = torch.device(device)
        self.asynchronous = bool(asynchronous)
        if self.device.type != "cuda":
            raise RuntimeError("n1b200 has no CPU path: NextDiTSystem1 needs device='cuda:N'")
        _lib.lib()
        self.num_inference_steps = num_inference_steps
        self.w = None

    # ------------------------------------------------------------------------------------------------ weights
    def load_state_dict(self, sd):
        from .manifest import nextdit_shapes
        want = nextdit_shapes(asynchronous=self.asynchronous)
        missing = [k for k in want if k not in sd and "mask_token" not in k and "visual_proj" not in k and "patch_embedder" not in k]
        if missing:
            raise KeyError("NextDiT state_dict misses %d tensors, e.g. %s" % (len(missing), missing[:3]))
        dev = self.device
        f32 = lambda k: sd[k].detach().to(dev, torch.float32).contiguous()
        b16 = lambda t: t.to(dev, torch.bfloat16).contiguous()
        w = {}
        for k in ("cond_projector.0", "cond_projector.2"):
            w[k + ".w"], w[k + ".b"] = b16(sd[k + ".weight"]), f32(k + ".bias")
        if self.asynchronous:
            self._load_rgb_branch(sd, w, f32, b16)
        self._load_dit(sd, w, f32, b16)
        self.w = w
        self._pos_cache = {}
        return self

    def _load_rgb_branch(self, sd, w, f32, b16):
        """DINOv2 ViT-S/14, MemoryEncoder and QFormer of the asynchronous head."""
        # DINOv2 ViT-S/14: im2col weight per channel with the ImageNet normalisation folded in
        Wpe, bpe = fold_patch_embed(f32("rgb_model.patch_embed.proj.weight"), f32("rgb_model.patch_embed.proj.bias"))
        w["vit.patch.w"], w["vit.patch.b"] = b16(Wpe), bpe
        pos = _resample_pos_embed(f32("rgb_model.pos_embed"))[0]
        w["vit.pos"] = pos[1:].contiguous()                                             # fp32 [256, 384]
        w["vit.cls"] = (f32("rgb_model.cls_token")[0, 0] + pos[0]).to(torch.bfloat16)    # cls token + its position
        for i in range(12):
            p, q = "rgb_model.blocks.%d." % i, "vit.%d." % i
            for n in ("norm1", "norm2"):
                w[q + n + ".w"], w[q + n + ".b"] = f32(p + n + ".weight"), f32(p + n + ".bias")
            for n in ("attn.qkv", "attn.proj", "mlp.fc1", "mlp.fc2"):
                w[q + n + ".w"], w[q + n + ".b"] = b16(sd[p + n + ".weight"]), f32(p + n + ".bias")
            w[q + "ls1"], w[q + "ls2"] = f32(p + "ls1.gamma"), f32(p + "ls2.gamma")
        w["vit.norm.w"], w["vit.norm.b"] = f32("rgb_model.norm.weight"), f32("rgb_model.norm.bias")
        # MemoryEncoder / QFormer (post-norm nn.Transformer layers)
        w["mem.pos"] = b16(sd["memory_encoder.memory_pos"])
        w["qf.query"] = b16(sd["rgb_resampler.query_tokens"].float() + sd["rgb_resampler.query_pos"].float())
        layers = [("memory_encoder.encoder.layers.%d." % i, "mem.%d." % i, False) for i in range(3)]
        layers += [("rgb_resampler.decoder.layers.%d." % i, "qf.%d." % i, True) for i in range(3)]
        for p, q, dec in layers:
            for a in ("self_attn", "multihead_attn") if dec else ("self_attn",):
                w[q + a + ".in.w"], w[q + a + ".in.b"] = b16(sd[p + a + ".in_proj_weight"]), f32(p + a + ".in_proj_bias")
                w[q + a + ".out.w"], w[q + a + ".out.b"] = b16(sd[p + a + ".out_proj.weight"]), f32(p + a + ".out_proj.bias")
            for n in ("linear1", "linear2"):
                w[q + n + ".w"], w[q + n + ".b"] = b16(sd[p + n + ".weight"]), f32(p + n + ".bias")
            for n in ("norm1", "norm2", "norm3") if dec else ("norm1", "norm2"):
                w[q + n + ".w"], w[q + n + ".b"] = f32(p + n + ".weight"), f32(p + n + ".bias")

    def _load_dit(self, sd, w, f32, b16):
        """Trajectory DiT, action encoder and decoder (both heads)."""
        dev = self.device
        p = "traj_dit.model."
        for n in ("caption_projection.linear_1", "caption_projection.linear_2", "time_caption_embed.timestep_embedder.linear_1",
                  "time_caption_embed.timestep_embedder.linear_2", "time_caption_embed.caption_embedder.1", "norm_out.linear_1"):
            w[n + ".w"], w[n + ".b"] = b16(sd[p + n + ".weight"]), f32(p + n + ".bias")
        w["cap_ln.w"], w["cap_ln.b"] = f32(p + "time_caption_embed.caption_embedder.0.weight"), f32(p + "time_caption_embed.caption_embedder.0.bias")
        mod_w, mod_b, kv_w = [], [], []
        for i in range(LAYERS):
            b, q = "%slayers.%d." % (p, i), "dit.%d." % i
            mod_w.append(sd[b + "norm1.linear.weight"].float())
            mod_b.append(sd[b + "norm1.linear.bias"].float())
            kv_w += list(fold_cross_kv(f32(b + "attn2.to_k.weight"), f32(b + "attn2.to_v.weight"),
                                       f32(b + "norm1_context.weight"), f32(b + "gate"), HD))
            w[q + "qkvq.w"] = b16(torch.cat([sd[b + "attn1.to_q.weight"], sd[b + "attn1.to_k.weight"],
                                             sd[b + "attn1.to_v.weight"], sd[b + "attn2.to_q.weight"]], dim=0).float())
            for a, n in (("attn1.norm_q", "nq1"), ("attn1.norm_k", "nk1"), ("attn2.norm_q", "nq2"), ("attn2.norm_k", "nk2")):
                w[q + n + ".w"], w[q + n + ".b"] = f32(b + a + ".weight"), f32(b + a + ".bias")
            w[q + "out.w"] = b16(sd[b + "attn2.to_out.0.weight"])
            l1, l3 = sd[b + "feed_forward.linear_1.weight"].float(), sd[b + "feed_forward.linear_3.weight"].float()
            w[q + "ff13.w"] = b16(torch.stack((l1, l3), dim=1).reshape(2 * FFN, DIM))  # rows (gate_j, up_j): SwiGLU epilogue
            w[q + "ff2.w"] = b16(sd[b + "feed_forward.linear_2.weight"])
            for a, n in (("norm1.norm", "n1"), ("norm2", "n2"), ("ffn_norm1", "f1"), ("ffn_norm2", "f2")):
                w[q + n] = f32(b + a + ".weight")
        w["dit.mod.w"], w["dit.mod.b"] = b16(torch.cat(mod_w, dim=0)), torch.cat(mod_b).to(dev).contiguous()
        w["dit.kv.w"] = b16(torch.cat(kv_w, dim=0))                                     # [12 * 768, 384]
        # norm_out.linear_2 followed by action_decoder: one [3 -> 8, 384] product
        Wh, bh = fold_head(f32(p + "norm_out.linear_2.weight"), f32(p + "norm_out.linear_2.bias"), f32("action_decoder.weight"),
                           f32("action_decoder.bias"))
        w["head.w"], w["head.b"] = b16(Wh), bh
        w["enc.w"], w["enc.b"] = f32("action_encoder.weight"), f32("action_encoder.bias")

    # ------------------------------------------------------------------------------------------------ building blocks
    def _lin(self, x, name, act=ACT_NONE, residual=None, gamma=None, bias=True):
        w = self.w
        return _lib.gemm(x, w[name + ".w"], bias=w[name + ".b"] if bias else None, act=act, residual=residual, gamma=gamma)

    def _ln(self, x, name, eps):
        return _lib.layernorm(x, self.w[name + ".w"], self.w[name + ".b"], eps)

    def _mha(self, q_in, kv_in, name, heads, batch, sq, sk):
        """nn.MultiheadAttention(batch_first=True), packed in_proj: rows [batch * s, D] -> out_proj(attention) + q_in."""
        D = q_in.shape[1]
        w = self.w
        if kv_in is q_in:
            qkv = _lib.gemm(q_in, w[name + ".in.w"], bias=w[name + ".in.b"])
            q, k, v = qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:]
        else:
            q = _lib.gemm(q_in, w[name + ".in.w"][:D], bias=w[name + ".in.b"][:D])
            kv = _lib.gemm(kv_in, w[name + ".in.w"][D:], bias=w[name + ".in.b"][D:])
            k, v = kv[:, :D], kv[:, D:]
        o = _lib.attention(q, k, v, heads, heads, D // heads, batch, sq, sk)
        return _lib.gemm(o, w[name + ".out.w"], bias=w[name + ".out.b"], residual=q_in)

    def _post_norm_layer(self, x, mem, q, heads, batch, sq, sk):
        """nn.TransformerEncoderLayer / DecoderLayer defaults (post-norm, ReLU, ff 2048, eps 1e-5)."""
        x = self._ln(self._mha(x, x, q + "self_attn", heads, batch, sq, sq), q + "norm1", 1e-5)
        n = 2
        if mem is not None:
            x = self._ln(self._mha(x, mem, q + "multihead_attn", heads, batch, sq, sk), q + "norm2", 1e-5)
            n = 3
        ff = self._lin(self._lin(x, q + "linear1", act=ACT_RELU), q + "linear2", residual=x)
        return self._ln(ff, q + "norm%d" % n, 1e-5)

    def _vit(self, frames):
        """frames fp32 [n, 224, 224, 3] in [0, 1] -> bf16 [n, 256, 384] (get_intermediate_layers(x)[0]: last block, final
        norm, class token dropped; dinov2.py L272-322)."""
        w, n = self.w, frames.shape[0]
        chans = [_bwd.patchify_depth(frames[..., c].contiguous()) for c in range(3)]       # 3 x [n * 256, 200]
        t = _lib.gemm(torch.cat(chans, dim=1), w["vit.patch.w"], bias=w["vit.patch.b"], out_fp32=True)
        t = (t.view(n, 256, DIM) + w["vit.pos"]).to(torch.bfloat16)
        t = torch.cat((w["vit.cls"].expand(n, 1, DIM), t), dim=1).reshape(n * 257, DIM)
        for i in range(12):
            q = "vit.%d." % i
            qkv = self._lin(self._ln(t, q + "norm1", 1e-6), q + "attn.qkv")
            o = _lib.attention(qkv[:, :DIM], qkv[:, DIM:2 * DIM], qkv[:, 2 * DIM:], HEADS, HEADS, HD, n, 257, 257)
            t = self._lin(o, q + "attn.proj", residual=t, gamma=w[q + "ls1"])
            h = self._lin(self._ln(t, q + "norm2", 1e-6), q + "mlp.fc1", act=ACT_GELU)
            t = self._lin(h, q + "mlp.fc2", residual=t, gamma=w[q + "ls2"])
        t = self._ln(t, "vit.norm", 1e-6)
        return t.view(n, 257, DIM)[:, 1:].contiguous()

    def condition_tokens(self, traj_latents, images_dp):
        """internvla_n1.py L363-382 per environment: -> bf16 [B, 36, 768]; the synchronous head: cond_projector(latents)
        alone, [B, n_query, 768] (images_dp is not read)."""
        assert self.w is not None, "load_state_dict first"
        B = traj_latents.shape[0]
        lat = traj_latents.to(self.device, torch.bfloat16).reshape(B * traj_latents.shape[1], -1).contiguous()
        lat = self._lin(self._lin(lat, "cond_projector.0", act=ACT_GELU_TANH), "cond_projector.2")
        if not self.asynchronous:
            return lat.view(B, -1, LATENT)
        img = images_dp.to(self.device, torch.float32)
        assert tuple(img.shape[1:]) == (2, 224, 224, 3), "images_dp is [B, 2, 224, 224, 3] ([pixel-goal frame, current frame])"
        feat = self._vit(img.reshape(B * 2, 224, 224, 3)).view(B, 512, DIM)
        x = (feat + self.w["mem.pos"][:512]).reshape(B * 512, DIM)
        for i in range(3):
            x = self._post_norm_layer(x, None, "mem.%d." % i, 6, B, 512, 512)
        mem = torch.cat((feat, x.view(B, 512, DIM)), dim=-1).reshape(B * 512, LATENT)
        q = self.w["qf.query"].unsqueeze(0).expand(B, -1, -1).reshape(B * 32, LATENT).contiguous()
        for i in range(3):
            q = self._post_norm_layer(q, mem, "qf.%d." % i, 12, B, 32, 512)
        return torch.cat((q.view(B, 32, LATENT), lat.view(B, -1, LATENT)), dim=1)

    # ------------------------------------------------------------------------------------------------ sampler
    def schedule(self, n=None):
        """FlowMatchEulerDiscreteScheduler().set_timesteps(n, sigmas=np.linspace(1, 1 / n, n)) (internvla_n1.py L395-396):
        -> (int64 timesteps [n], float32 sigmas [n + 1])."""
        return flow_match_schedule(n or self.num_inference_steps)

    def _pos(self, T):
        """SinusoidalPositionalEncoding(384) of arange(T) (internvla_n1_arch.py L52-73), fp32 [T, 384]."""
        if T not in self._pos_cache:
            half = DIM // 2
            freqs = torch.arange(T, dtype=torch.float32)[:, None] * torch.exp(
                -torch.arange(half, dtype=torch.float) * (torch.log(torch.tensor(10000.0)) / half))[None, :]
            self._pos_cache[T] = torch.cat((torch.sin(freqs), torch.cos(freqs)), dim=-1).to(self.device).contiguous()
        return self._pos_cache[T]

    def _time_freqs(self, timesteps):
        """Timesteps(256, flip_sin_to_cos=True, downscale_freq_shift=0) of the schedule, bf16 on the device (cached: a host
        table cannot be uploaded while a CUDA graph is being captured)."""
        key = tuple(int(t) for t in timesteps)
        if key not in self._pos_cache:
            half = 128
            freq = torch.exp(-math.log(10000) * torch.arange(half, dtype=torch.float32) / half)
            ang = timesteps.float()[:, None] * freq[None, :]
            self._pos_cache[key] = torch.cat((torch.cos(ang), torch.sin(ang)), dim=-1).to(self.device, torch.bfloat16)
        return self._pos_cache[key]

    def _conditioning(self, z, timesteps):
        """Everything the 12 blocks read that does not depend on the trajectories.  z bf16 [G, 36, 768]."""
        w, G, S = self.w, z.shape[0], len(timesteps)
        enc = self._lin(self._lin(z.reshape(G * z.shape[1], LATENT), "caption_projection.linear_1", act=ACT_GELU_TANH),
                        "caption_projection.linear_2")                                           # [G * 36, 384]
        pool = enc.view(G, -1, DIM).float().mean(dim=1).to(torch.bfloat16)                        # all-ones caption mask
        ce = self._lin(_lib.layernorm(pool, w["cap_ln.w"], w["cap_ln.b"], 1e-5), "time_caption_embed.caption_embedder.1")
        tf = self._time_freqs(timesteps)                                                          # [S, 256]
        te = self._lin(self._lin(tf, "time_caption_embed.timestep_embedder.linear_1", act=ACT_SILU),
                       "time_caption_embed.timestep_embedder.linear_2")                          # [S, 384]
        st = F.silu(te[:, None, :] + ce[None, :, :]).reshape(S * G, DIM).contiguous()             # silu(temb), S * G rows
        mods = _lib.gemm(st, w["dit.mod.w"], bias=w["dit.mod.b"]).view(S, G, LAYERS, 4 * DIM)
        scale_out = self._lin(st, "norm_out.linear_1").view(S, G, DIM)
        e = _lib.mod_norm(enc, None, None, 1, 1e-5, MOD_RMS_SCALE)                                # RMSNorm, weight folded
        kv = _lib.gemm(e, w["dit.kv.w"])                                                          # [G * 36, 12 * 768]
        kn = torch.empty(e.shape[0], LAYERS * DIM, device=self.device, dtype=torch.bfloat16)
        for l in range(LAYERS):
            _lib.layernorm(kv[:, l * 2 * DIM:l * 2 * DIM + DIM], w["dit.%d.nk2.w" % l], w["dit.%d.nk2.b" % l], 1e-5,
                           out=kn[:, l * DIM:(l + 1) * DIM])
        return mods, scale_out, kn, kv

    def _dit_step(self, x, mods_i, scale_out_i, kn, kv, rows_per_group, n_seq, T, Sk, kv_div):
        """One evaluation of the 12 blocks + norm_out + action_decoder on rows x [n_seq * T, 384] -> bf16 [rows, 8]."""
        w = self.w
        for l in range(LAYERS):
            q = "dit.%d." % l
            m = mods_i[:, l]                                                       # [G, 1536] view: scale_msa | gate_msa | scale_mlp | gate_mlp
            h = _lib.mod_norm(x, w[q + "n1"], m[:, :DIM], rows_per_group, 1e-5, MOD_RMS_SCALE)
            p = _lib.gemm(h, w[q + "qkvq.w"])                                       # self q | k | v | cross q
            q1 = _lib.layernorm(p[:, :DIM], w[q + "nq1.w"], w[q + "nq1.b"], 1e-5)
            k1 = _lib.layernorm(p[:, DIM:2 * DIM], w[q + "nk1.w"], w[q + "nk1.b"], 1e-5)
            q2 = _lib.layernorm(p[:, 3 * DIM:], w[q + "nq2.w"], w[q + "nq2.b"], 1e-5)
            o_self = _lib.attention(q1, k1, p[:, 2 * DIM:3 * DIM], HEADS, HEADS, HD, n_seq, T, T)
            o_cross = _lib.attention(q2, kn[:, l * DIM:(l + 1) * DIM], kv[:, l * 2 * DIM + DIM:(l + 1) * 2 * DIM], HEADS, HEADS, HD,
                                     n_seq, T, Sk, kv_div=kv_div)                  # tanh(gate) is folded into V
            hid = _lib.gemm(_lib.add(o_self, o_cross), w[q + "out.w"])
            x = _lib.mod_norm(hid, w[q + "n2"], m[:, DIM:2 * DIM], rows_per_group, 1e-5, MOD_GATED_RESIDUAL, residual=x)
            h = _lib.mod_norm(x, w[q + "f1"], m[:, 2 * DIM:3 * DIM], rows_per_group, 1e-5, MOD_RMS_SCALE)
            f = _lib.gemm(_lib.gemm(h, w[q + "ff13.w"], act=ACT_SWIGLU), w[q + "ff2.w"])
            x = _lib.mod_norm(f, w[q + "f2"], m[:, 3 * DIM:], rows_per_group, 1e-5, MOD_GATED_RESIDUAL, residual=x)
        y = _lib.mod_norm(x, None, scale_out_i, rows_per_group, 1e-6, MOD_LN_SCALE)
        return _lib.gemm(y, w["head.w"], bias=w["head.b"])

    def sample(self, cond_tokens, x_init, guidance_scale=1.0, num_inference_steps=None, num_sample_trajs=32, exact_cfg=False,
               graph=None):
        """The denoising loop of internvla_n1.py L383-428.  cond_tokens bf16 [B, 36, 768]; x_init [B * Ns, T, 3] (the
        reference draws it with randn_tensor in the model dtype) -> fp32 [B * Ns, T, 3] holding bf16-representable values.
        `graph` (default on): the ~5 700 launches of a call are replayed from a CUDA graph cached per problem shape --
        issued one ctypes call at a time the loop is host-bound (17 us per launch against ~10 us of kernel)."""
        if graph is None:
            graph = not torch.cuda.is_current_stream_capturing()
        if not graph:
            return self._sample_eager(cond_tokens, x_init, guidance_scale, num_inference_steps, num_sample_trajs, exact_cfg)
        dev = self.device
        num_inference_steps = num_inference_steps or self.num_inference_steps
        key = (tuple(cond_tokens.shape), tuple(x_init.shape), float(guidance_scale), num_inference_steps, num_sample_trajs,
               bool(exact_cfg))
        if not hasattr(self, "_graphs"):
            self._graphs = {}
        hit = self._graphs.get(key)
        if hit is None:
            st = dict(cond=torch.empty(cond_tokens.shape, device=dev, dtype=torch.bfloat16),
                      x0=torch.empty(x_init.shape, device=dev, dtype=torch.bfloat16))
            st["cond"].copy_(cond_tokens), st["x0"].copy_(x_init)
            args = (guidance_scale, num_inference_steps, num_sample_trajs, exact_cfg)
            side = torch.cuda.Stream(device=dev)
            side.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(side):
                self._sample_eager(st["cond"], st["x0"], *args)     # warm-up: cached tables, allocator state of `side`
                side.synchronize()
                before = _lib.prof_read()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, stream=side, capture_error_mode="thread_local"):
                    out = self._sample_eager(st["cond"], st["x0"], *args)
                nodes = _lib.prof_read()                             # kernels in the graph = launches of every replay
                _lib.lib().n1_prof_add(before["gemm_launches"], before["total_launches"])
            torch.cuda.current_stream(dev).wait_stream(side)
            hit = self._graphs[key] = (g, st, out, nodes)
        g, st, out, nodes = hit
        st["cond"].copy_(cond_tokens, non_blocking=True)
        st["x0"].copy_(x_init, non_blocking=True)
        g.replay()
        _lib.lib().n1_prof_add(nodes["gemm_launches"], nodes["total_launches"])
        return out.clone()

    def _sample_eager(self, cond_tokens, x_init, guidance_scale, num_inference_steps, num_sample_trajs, exact_cfg):
        B, Sk = cond_tokens.shape[0], cond_tokens.shape[1]
        Ns, T = num_sample_trajs, x_init.shape[1]
        assert x_init.shape[0] == B * Ns and x_init.shape[2] == 3
        cfg = exact_cfg or float(guidance_scale) != 1.0
        z = cond_tokens.to(self.device, torch.bfloat16).contiguous()
        if cfg:
            z = torch.cat((torch.zeros_like(z), z), dim=0)                          # [null | conditional] halves
        timesteps, sigmas = self.schedule(num_inference_steps)
        mods, scale_out, kn, kv = self._conditioning(z, timesteps)
        lat = x_init.to(self.device, torch.bfloat16).float().contiguous()           # model-dtype values, fp32 storage
        n_rows = B * Ns * T
        halves = 2 if cfg else 1
        x = torch.empty(halves * n_rows, DIM, device=self.device, dtype=torch.bfloat16)
        pos = self._pos(T)
        for i in range(len(timesteps)):
            for h in range(halves):                                                 # latent_features.repeat(2, 1, 1)
                _lib.action_embed(lat, self.w["enc.w"], self.w["enc.b"], pos, out=x[h * n_rows:(h + 1) * n_rows])
            pred = self._dit_step(x, mods[i], scale_out[i], kn, kv, Ns * T, halves * B * Ns, T, Sk, Ns)
            _lib.cfg_euler(pred, n_rows, cfg, guidance_scale, float(sigmas[i + 1] - sigmas[i]), lat)
        return lat.view(B * Ns, T, 3)

    def generate_traj(self, traj_latents, images_dp, depths_dp=None, predict_step_nums=32, guidance_scale=1.0,
                      num_inference_steps=10, num_sample_trajs=32, x_init=None, exact_cfg=False, graph=None):
        """Signature of the reference's generate_traj (depths_dp is unused by this System 1, images_dp by the synchronous
        head).  `x_init` injects the initial
        noise (tests); by default it is drawn on the device in the latents' dtype as the reference does."""
        B = traj_latents.shape[0]
        if x_init is None:
            x_init = torch.randn(B * num_sample_trajs, predict_step_nums, 3, device=self.device, dtype=torch.bfloat16)
        cond = self.condition_tokens(traj_latents, images_dp)
        out = self.sample(cond, x_init, guidance_scale, num_inference_steps, num_sample_trajs, exact_cfg, graph=graph)
        return out.to(traj_latents.dtype if traj_latents.is_floating_point() else torch.bfloat16)
