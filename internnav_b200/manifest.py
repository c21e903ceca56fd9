"""Parameter manifest of the System-1 head: names and shapes exactly as `NavDP_Policy_DPT_CriticSum_DAT.state_dict()`
produces them in the reference (navdp.py L16-114; SURVEY.md Appendix A), generated from the dimensions -- so the mirror
class can be random-initialised, checkpointed and handed to an optimiser without the reference installed.
tests/test_manifest.py checks it against the manifest dumped from the reference class itself.
"""
from collections import OrderedDict

import torch


def _mha(p, D):
    return [(p + "in_proj_weight", (3 * D, D)), (p + "in_proj_bias", (3 * D,)), (p + "out_proj.weight", (D, D)),
            (p + "out_proj.bias", (D,))]


def _dec_layer(p, D, ff):
    out = _mha(p + "self_attn.", D) + _mha(p + "multihead_attn.", D)
    out += [(p + "linear1.weight", (ff, D)), (p + "linear1.bias", (ff,)), (p + "linear2.weight", (D, ff)),
            (p + "linear2.bias", (D,))]
    for n in ("norm1", "norm2", "norm3"):
        out += [(p + n + ".weight", (D,)), (p + n + ".bias", (D,))]
    return out


def _vit(p, D=384, depth=12, grid=37):
    out = [(p + "cls_token", (1, 1, D)), (p + "pos_embed", (1, grid * grid + 1, D)), (p + "mask_token", (1, D)),
           (p + "patch_embed.proj.weight", (D, 3, 14, 14)), (p + "patch_embed.proj.bias", (D,))]
    for i in range(depth):
        b = "%sblocks.%d." % (p, i)
        out += [(b + "norm1.weight", (D,)), (b + "norm1.bias", (D,)), (b + "attn.qkv.weight", (3 * D, D)),
                (b + "attn.qkv.bias", (3 * D,)), (b + "attn.proj.weight", (D, D)), (b + "attn.proj.bias", (D,)),
                (b + "ls1.gamma", (D,)), (b + "norm2.weight", (D,)), (b + "norm2.bias", (D,)),
                (b + "mlp.fc1.weight", (4 * D, D)), (b + "mlp.fc1.bias", (4 * D,)), (b + "mlp.fc2.weight", (D, 4 * D)),
                (b + "mlp.fc2.bias", (D,)), (b + "ls2.gamma", (D,))]
    out += [(p + "norm.weight", (D,)), (p + "norm.bias", (D,))]
    return out


def navdp_shapes(memory_size=2, predict_size=32, temporal_depth=16, token_dim=384, vlm_token_dim=3584,
                 navdp_version=0.1):
    D = token_dim
    items = [("cond_pos_embed", (1, memory_size * 16 + 2, D)), ("out_pos_embed", (1, predict_size, D))]
    items += _vit("rgbd_encoder.rgb_model.") + _vit("rgbd_encoder.depth_model.")
    pe_rows = (memory_size * 2) * 256 if navdp_version > 0.0 else (memory_size + 1) * 256
    items += [("rgbd_encoder.former_query.weight", (memory_size * 16, D)), ("rgbd_encoder.former_pe.weight", (pe_rows, D))]
    for i in range(2):
        items += _dec_layer("rgbd_encoder.former_net.layers.%d." % i, D, 2048)
    items += [("rgbd_encoder.project_layer.weight", (D, D)), ("rgbd_encoder.project_layer.bias", (D,)),
              ("point_encoder.weight", (D, 3)), ("point_encoder.bias", (D,))]
    items += _dec_layer("decoder_layer.", D, 4 * D)
    for i in range(temporal_depth):
        items += _dec_layer("decoder.layers.%d." % i, D, 4 * D)
    items += [("input_embed.weight", (D, 3)), ("input_embed.bias", (D,)), ("layernorm.weight", (D,)),
              ("layernorm.bias", (D,)), ("action_head.weight", (3, D)), ("action_head.bias", (3,)),
              ("critic_head.weight", (1, D)), ("critic_head.bias", (1,))]
    v = vlm_token_dim
    for idx, (o, i) in zip((0, 2, 4), ((v // 4, v), (v // 8, v // 4), (D, v // 8))):
        items += [("vlm_embed_mlp.%d.weight" % idx, (o, i)), ("vlm_embed_mlp.%d.bias" % idx, (o,))]
    g = "goal_compressor."
    items += [(g + "target_embedding.weight", (1, D)), (g + "positional_encoding.pe", (1000, D)),
              (g + "token_positional_encoding.position_embedding.weight", (5000, D)),
              (g + "query_positional_encoding.position_embedding.weight", (5000, D))]
    items += _mha(g + "cross_attention.", D)
    for idx, (o, i) in zip((0, 2), ((D // 2, 2), (D, D // 2))):
        items += [("pg_embed_mlp.%d.weight" % idx, (o, i)), ("pg_embed_mlp.%d.bias" % idx, (o,))]
    for idx, (o, i) in zip((0, 2, 4), ((D // 2, D), (D // 4, D // 2), (2, D // 4))):
        items += [("pg_pred_mlp.%d.weight" % idx, (o, i)), ("pg_pred_mlp.%d.bias" % idx, (o,))]
    return OrderedDict(items)


def navdp_policy_shapes(memory_size=8, predict_size=24, temporal_depth=16, token_dim=384):
    """Inference-relevant tensors of the stand-alone NavDPNet (navdp_policy.py L62-134; the image / pixel goal encoders and
    auxiliary heads, which only `forward` (training) reads, are left out), under the reference's state_dict names."""
    D = token_dim
    items = _vit("rgbd_encoder.rgb_model.") + _vit("rgbd_encoder.depth_model.")
    items += [("rgbd_encoder.former_query.position_embedding.weight", (memory_size * 16, D)),
              ("rgbd_encoder.former_pe.position_embedding.weight", ((memory_size + 1) * 256, D))]
    for i in range(2):
        items += _dec_layer("rgbd_encoder.former_net.layers.%d." % i, D, 2048)
    items += [("rgbd_encoder.project_layer.weight", (D, D)), ("rgbd_encoder.project_layer.bias", (D,)),
              ("point_encoder.weight", (D, 3)), ("point_encoder.bias", (D,))]
    for i in range(temporal_depth):
        items += _dec_layer("decoder.layers.%d." % i, D, 4 * D)
    items += [("input_embed.weight", (D, 3)), ("input_embed.bias", (D,)),
              ("cond_pos_embed.position_embedding.weight", (memory_size * 16 + 4, D)),
              ("out_pos_embed.position_embedding.weight", (predict_size, D)),
              ("layernorm.weight", (D,)), ("layernorm.bias", (D,)), ("action_head.weight", (3, D)), ("action_head.bias", (3,)),
              ("critic_head.weight", (1, D)), ("critic_head.bias", (1,))]
    return OrderedDict(items)


def random_navdp_policy_state_dict(seed=0, device="cpu", dtype=torch.float32, **dims):
    """Seeded random weights of the stand-alone NavDPNet shapes (same scaling rules as random_navdp_state_dict)."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    out = OrderedDict()
    for name, shape in navdp_policy_shapes(**dims).items():
        last = name.split(".")[-1]
        if (("norm" in name and last == "weight") or last == "gamma") and len(shape) == 1:
            t = 1.0 + 0.1 * torch.randn(shape, generator=g)
        elif "position_embedding" in name or "pos_embed" in name or "cls_token" in name or "mask_token" in name:
            t = 0.1 * torch.randn(shape, generator=g)
        elif len(shape) >= 2:
            fan_in = 1
            for s in shape[1:]:
                fan_in *= s
            t = torch.randn(shape, generator=g) / fan_in ** 0.5
        else:
            t = 0.02 * torch.randn(shape, generator=g)
        out[name] = t.to(device=device, dtype=dtype)
    return out


def random_navdp_state_dict(seed=0, device="cpu", dtype=torch.float32, **dims):
    """Random weights of the right shapes (synthetic benchmark / smoke runs; there are no checkpoints offline).
    Scales keep activations O(1); tables the reference zero-initialises get small non-zero values."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    out = OrderedDict()
    for name, shape in navdp_shapes(**dims).items():
        last = name.split(".")[-1]
        if (("norm" in name and last == "weight") or last == "gamma") and len(shape) == 1:
            t = 1.0 + 0.1 * torch.randn(shape, generator=g)
        elif len(shape) >= 2 and last not in ("pe",) and "embed" not in last and "token" not in last and "former" not in name \
                and "position_embedding" not in name and "target_embedding" not in name:
            fan_in = 1
            for s in shape[1:]:
                fan_in *= s
            t = torch.randn(shape, generator=g) / fan_in ** 0.5
        elif len(shape) >= 2:
            t = 0.1 * torch.randn(shape, generator=g)
        else:
            t = 0.02 * torch.randn(shape, generator=g)
        out[name] = t.to(device=device, dtype=dtype)
    return out


# ---------------------------------------------------------------------------------------------- NextDiT System 1 (f1)
def _enc_layer(p, D, ff):
    out = _mha(p + "self_attn.", D)
    out += [(p + "linear1.weight", (ff, D)), (p + "linear1.bias", (ff,)), (p + "linear2.weight", (D, ff)),
            (p + "linear2.bias", (D,))]
    for n in ("norm1", "norm2"):
        out += [(p + n + ".weight", (D,)), (p + n + ".bias", (D,))]
    return out


NEXTDIT_ASYNC_ONLY = ("rgb_model.", "memory_encoder.", "rgb_resampler.")


def nextdit_shapes(dim=384, layers=12, heads=6, latent=768, vlm_token_dim=3584, ffn=1024, asynchronous=True):
    """Tensors of the `nextdit_async` System 1 under the reference's attribute paths below `InternVLAN1ForCausalLM.model`
    (internvla_n1_arch.py L131-145: cond_projector, rgb_model, memory_encoder, rgb_resampler, action_encoder / decoder,
    traj_dit = NextDiTCrossAttn(latent_embedding_size=768), nextdit_crossattn_traj.py L46-82).  `asynchronous=False`:
    the synchronous `nextdit` head, which has no rgb_model / memory_encoder / rgb_resampler (L141-145)."""
    if not asynchronous:
        full = nextdit_shapes(dim, layers, heads, latent, vlm_token_dim, ffn)
        return OrderedDict((k, v) for k, v in full.items() if not k.startswith(NEXTDIT_ASYNC_ONLY))
    D, L = dim, latent
    items = [("cond_projector.0.weight", (L, vlm_token_dim)), ("cond_projector.0.bias", (L,)),
             ("cond_projector.2.weight", (L, L)), ("cond_projector.2.bias", (L,))]
    items += _vit("rgb_model.")
    items += [("memory_encoder.memory_pos", (512, D))]
    for i in range(3):
        items += _enc_layer("memory_encoder.encoder.layers.%d." % i, D, 2048)
    items += [("rgb_resampler.query_tokens", (32, L)), ("rgb_resampler.query_pos", (32, L))]
    for i in range(3):
        items += _dec_layer("rgb_resampler.decoder.layers.%d." % i, L, 2048)
    items += [("rgb_resampler.visual_proj.weight", (L, L)), ("rgb_resampler.visual_proj.bias", (L,)),
              ("action_encoder.weight", (D, 3)), ("action_encoder.bias", (D,)),
              ("action_decoder.weight", (3, D)), ("action_decoder.bias", (3,))]
    p = "traj_dit.model."
    items += [(p + "caption_projection.linear_1.weight", (D, L)), (p + "caption_projection.linear_1.bias", (D,)),
              (p + "caption_projection.linear_2.weight", (D, D)), (p + "caption_projection.linear_2.bias", (D,)),
              (p + "patch_embedder.proj.weight", (D, D)), (p + "patch_embedder.proj.bias", (D,)),
              (p + "time_caption_embed.timestep_embedder.linear_1.weight", (D, 256)),
              (p + "time_caption_embed.timestep_embedder.linear_1.bias", (D,)),
              (p + "time_caption_embed.timestep_embedder.linear_2.weight", (D, D)),
              (p + "time_caption_embed.timestep_embedder.linear_2.bias", (D,)),
              (p + "time_caption_embed.caption_embedder.0.weight", (D,)), (p + "time_caption_embed.caption_embedder.0.bias", (D,)),
              (p + "time_caption_embed.caption_embedder.1.weight", (D, D)), (p + "time_caption_embed.caption_embedder.1.bias", (D,))]
    for i in range(layers):
        b = "%slayers.%d." % (p, i)
        items += [(b + "gate", (heads,))]
        for a in ("attn1.", "attn2."):
            items += [(b + a + "to_q.weight", (D, D)), (b + a + "to_k.weight", (D, D)), (b + a + "to_v.weight", (D, D)),
                      (b + a + "norm_q.weight", (D,)), (b + a + "norm_q.bias", (D,)), (b + a + "norm_k.weight", (D,)),
                      (b + a + "norm_k.bias", (D,))]
        items += [(b + "attn2.to_out.0.weight", (D, D)), (b + "feed_forward.linear_1.weight", (ffn, D)),
                  (b + "feed_forward.linear_2.weight", (D, ffn)), (b + "feed_forward.linear_3.weight", (ffn, D)),
                  (b + "norm1.linear.weight", (4 * D, D)), (b + "norm1.linear.bias", (4 * D,)), (b + "norm1.norm.weight", (D,)),
                  (b + "ffn_norm1.weight", (D,)), (b + "norm2.weight", (D,)), (b + "ffn_norm2.weight", (D,)),
                  (b + "norm1_context.weight", (D,))]
    items += [(p + "norm_out.linear_1.weight", (D, D)), (p + "norm_out.linear_1.bias", (D,)),
              (p + "norm_out.linear_2.weight", (D, D)), (p + "norm_out.linear_2.bias", (D,))]
    return OrderedDict(items)


def random_nextdit_state_dict(seed=0, device="cpu", dtype=torch.float32, **dims):
    """Seeded random weights of the NextDiT System-1 shapes.  The reference zero-initialises `gate` (tanh(0) = 0 would
    switch the cross-attention off): it gets O(0.5) values here so that branch is exercised."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    out = OrderedDict()
    for name, shape in nextdit_shapes(**dims).items():
        last = name.split(".")[-1]
        if last == "gate":
            t = 0.5 * torch.randn(shape, generator=g)
        elif len(shape) == 1 and last in ("weight", "gamma") and ("norm" in name or "caption_embedder.0" in name or last == "gamma"):
            t = 1.0 + 0.1 * torch.randn(shape, generator=g)
        elif "pos_embed" in name or "cls_token" in name or "mask_token" in name:
            t = 0.1 * torch.randn(shape, generator=g)
        elif last in ("memory_pos", "query_tokens", "query_pos"):
            t = 0.5 * torch.randn(shape, generator=g)
        elif len(shape) >= 2:
            fan_in = 1
            for s in shape[1:]:
                fan_in *= s
            t = torch.randn(shape, generator=g) / fan_in ** 0.5
        else:
            t = 0.02 * torch.randn(shape, generator=g)
        out[name] = t.to(device=device, dtype=dtype)
    return out


# ---------------------------------------------------------------------------------------------- System 2
def s2_shapes(cfg, lm_head=False):
    """Qwen2.5-VL parameter names/shapes in the transformers==4.51 checkpoint layout the reference loads, plus
    InternVLA-N1's `model.latent_queries` (internvla_n1_arch.py L123).  `lm_head=True` adds the untied output projection
    that only the greedy decode reads."""
    Hv, H = cfg["v_hidden"], cfg["hidden"]
    unit = cfg["v_merge"] ** 2
    out = [("visual.patch_embed.proj.weight", (Hv, 3, cfg["v_tpatch"], cfg["v_patch"], cfg["v_patch"]))]
    for i in range(cfg["v_depth"]):
        b = "visual.blocks.%d." % i
        out += [(b + "norm1.weight", (Hv,)), (b + "norm2.weight", (Hv,)), (b + "attn.qkv.weight", (3 * Hv, Hv)),
                (b + "attn.qkv.bias", (3 * Hv,)), (b + "attn.proj.weight", (Hv, Hv)), (b + "attn.proj.bias", (Hv,)),
                (b + "mlp.gate_proj.weight", (cfg["v_inter"], Hv)), (b + "mlp.gate_proj.bias", (cfg["v_inter"],)),
                (b + "mlp.up_proj.weight", (cfg["v_inter"], Hv)), (b + "mlp.up_proj.bias", (cfg["v_inter"],)),
                (b + "mlp.down_proj.weight", (Hv, cfg["v_inter"])), (b + "mlp.down_proj.bias", (Hv,))]
    out += [("visual.merger.ln_q.weight", (Hv,)), ("visual.merger.mlp.0.weight", (Hv * unit, Hv * unit)),
            ("visual.merger.mlp.0.bias", (Hv * unit,)), ("visual.merger.mlp.2.weight", (cfg["v_out"], Hv * unit)),
            ("visual.merger.mlp.2.bias", (cfg["v_out"],))]
    out += [("model.embed_tokens.weight", (cfg["vocab"], H)), ("model.latent_queries", (1, cfg["n_query"], H))]
    qd, kd = cfg["heads"] * cfg["head_dim"], cfg["kv_heads"] * cfg["head_dim"]
    for i in range(cfg["layers"]):
        b = "model.layers.%d." % i
        out += [(b + "input_layernorm.weight", (H,)), (b + "post_attention_layernorm.weight", (H,)),
                (b + "self_attn.q_proj.weight", (qd, H)), (b + "self_attn.q_proj.bias", (qd,)),
                (b + "self_attn.k_proj.weight", (kd, H)), (b + "self_attn.k_proj.bias", (kd,)),
                (b + "self_attn.v_proj.weight", (kd, H)), (b + "self_attn.v_proj.bias", (kd,)),
                (b + "self_attn.o_proj.weight", (H, qd)), (b + "mlp.gate_proj.weight", (cfg["inter"], H)),
                (b + "mlp.up_proj.weight", (cfg["inter"], H)), (b + "mlp.down_proj.weight", (H, cfg["inter"]))]
    out += [("model.norm.weight", (H,))]
    if lm_head:
        out += [("lm_head.weight", (cfg["vocab"], H))]
    return OrderedDict(out)


def random_s2_state_dict(cfg, seed=0, device="cuda", dtype=torch.bfloat16, lm_head=False):
    """Random Qwen2.5-VL-shaped weights generated directly on `device` (synthetic benchmark runs; no checkpoints are
    available offline).  Norm weights ~1, matrices ~N(0, 1/fan_in), embeddings ~N(0, 1)."""
    g = torch.Generator(device=device).manual_seed(seed)
    out = OrderedDict()
    for name, shape in s2_shapes(cfg, lm_head=lm_head).items():
        if name.endswith("norm1.weight") or name.endswith("norm2.weight") or name.endswith("layernorm.weight") \
                or name.endswith("norm.weight") or name.endswith("ln_q.weight"):
            t = 1.0 + 0.1 * torch.randn(shape, generator=g, device=device)
        elif name.endswith(".bias"):
            t = 0.02 * torch.randn(shape, generator=g, device=device)
        elif name in ("model.embed_tokens.weight", "model.latent_queries"):
            t = torch.randn(shape, generator=g, device=device, dtype=dtype)
        else:
            fan_in = 1
            for s in shape[1:]:
                fan_in *= s
            t = torch.randn(shape, generator=g, device=device, dtype=dtype) / fan_in ** 0.5
        out[name] = t.to(dtype)
    return out
