"""BASELINE ARM of bench.py, not the product and not the parity oracle: the reference algorithm as BATCHED eager PyTorch
on the GPU -- bf16, every Linear through cuBLAS (F.linear), every attention through F.scaled_dot_product_attention
(flash / memory-efficient kernels), B environments per call.  This is the "PyTorch-eager on the same H100 at batch 64"
denominator of north_star's >= 10x target and the honest kernel-level comparison for the n1b200 path (VERDICT r1, measurement
item b): same shapes, same batch, library kernels instead of ours.

The System-2 functions restate oracle/qwen_oracle.py (itself pinned to transformers' Qwen2.5-VL blocks) for a batch of
equal-length prompts with one image each (the benchmark shape); tests/test_eager_gpu_gpu.py checks them against that
oracle.  System 1 runs oracle/navdp_oracle.py with its attention switched to SDPA.
"""
import torch
import torch.nn.functional as F

from . import navdp_oracle as O, qwen_oracle as Q


def _rms(x, w, eps):
    v = x.float()
    return (v * torch.rsqrt(v.pow(2).mean(-1, keepdim=True) + eps)).to(x.dtype) * w.to(x.dtype)


def _rot_half(x):
    h = x.shape[-1] // 2
    return torch.cat((-x[..., h:], x[..., :h]), dim=-1)


def vit_forward_batched(sd, cfg, pixel_values, grid, B, p="visual."):
    """B images of the same grid: [B * N, 1176] -> [B * N / 4, v_out].  Window attention: the windows of one image are
    grouped by length (64 / 32 / 16 tokens for a 28 x 28 grid) and every group is one batched SDPA call."""
    Hv, heads, unit = cfg["v_hidden"], cfg["v_heads"], cfg["v_merge"] ** 2
    hd = Hv // heads
    dt = pixel_values.dtype
    dev = pixel_values.device
    pos_ids, window_index, cu_window, cu_full = Q.vit_indices([grid], cfg["v_merge"], cfg["v_patch"], cfg["v_window"])
    N = grid[0] * grid[1] * grid[2]
    x = F.linear(pixel_values, sd[p + "patch_embed.proj.weight"].reshape(Hv, -1).to(dt)).view(B, N, Hv)
    dim = hd // 2
    inv_freq = 1.0 / (10000.0 ** (torch.arange(0, dim, 2, dtype=torch.float, device=dev) / dim))
    freqs = torch.outer(torch.arange(int(max(grid[1], grid[2])), device=dev, dtype=torch.float), inv_freq)
    rot = freqs[pos_ids.to(dev)].flatten(1)
    widx = window_index.to(dev)
    x = x.reshape(B, N // unit, unit, Hv)[:, widx].reshape(B, N, Hv)
    rot = rot.reshape(N // unit, unit, -1)[widx].reshape(N, -1)
    emb = torch.cat((rot, rot), dim=-1)
    cos, sin = emb.cos()[None, :, None, :], emb.sin()[None, :, None, :]
    lens = (cu_window[1:] - cu_window[:-1]).tolist()
    starts = cu_window[:-1].tolist()
    groups = {}
    for s0, L in zip(starts, lens):
        groups.setdefault(L, []).append(s0)
    gidx = {L: (torch.tensor(st, device=dev)[:, None] + torch.arange(L, device=dev)[None, :]) for L, st in groups.items()}
    for l in range(cfg["v_depth"]):
        b = "%sblocks.%d." % (p, l)
        h = _rms(x, sd[b + "norm1.weight"], 1e-6)
        qkv = F.linear(h, sd[b + "attn.qkv.weight"].to(dt), sd[b + "attn.qkv.bias"].to(dt)).view(B, N, 3, heads, hd)
        q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
        q = (q.float() * cos + _rot_half(q.float()) * sin).to(dt)
        k = (k.float() * cos + _rot_half(k.float()) * sin).to(dt)
        if l in cfg["fullatt"]:
            a = F.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2)).transpose(1, 2)
        else:
            a = torch.empty_like(q)
            for L, idx in gidx.items():
                nw = idx.shape[0]
                qq, kk, vv = (t[:, idx].reshape(B * nw, L, heads, hd).transpose(1, 2) for t in (q, k, v))
                o = F.scaled_dot_product_attention(qq, kk, vv).transpose(1, 2).reshape(B, nw, L, heads, hd)
                a[:, idx] = o
        x = x + F.linear(a.reshape(B, N, Hv), sd[b + "attn.proj.weight"].to(dt), sd[b + "attn.proj.bias"].to(dt))
        h = _rms(x, sd[b + "norm2.weight"], 1e-6)
        g = F.linear(h, sd[b + "mlp.gate_proj.weight"].to(dt), sd[b + "mlp.gate_proj.bias"].to(dt))
        u = F.linear(h, sd[b + "mlp.up_proj.weight"].to(dt), sd[b + "mlp.up_proj.bias"].to(dt))
        x = x + F.linear(F.silu(g) * u, sd[b + "mlp.down_proj.weight"].to(dt), sd[b + "mlp.down_proj.bias"].to(dt))
    m = _rms(x, sd[p + "merger.ln_q.weight"], 1e-6).view(B, N // unit, Hv * unit)
    m = F.linear(F.gelu(F.linear(m, sd[p + "merger.mlp.0.weight"].to(dt), sd[p + "merger.mlp.0.bias"].to(dt))),
                 sd[p + "merger.mlp.2.weight"].to(dt), sd[p + "merger.mlp.2.bias"].to(dt))
    return m[:, torch.argsort(widx)].reshape(B * (N // unit), -1)


def text_forward_batched(sd, cfg, x, position_ids, p="model."):
    """[B, S, H] + position ids [3, B, S] -> final-norm hidden states; causal GQA attention through SDPA."""
    dt = x.dtype
    B, S, H = x.shape
    heads, kvh, hd = cfg["heads"], cfg["kv_heads"], cfg["head_dim"]
    inv_freq = 1.0 / (cfg["rope_theta"] ** (torch.arange(0, hd, 2, dtype=torch.int64, device=x.device).float() / hd))
    freqs = position_ids[:, :, :, None].float() * inv_freq[None, None, None, :]
    emb = torch.cat((freqs, freqs), dim=-1)
    cos, sin = emb.cos().to(dt), emb.sin().to(dt)
    sec = cfg["mrope"] * 2
    cos = torch.cat([m[i % 3] for i, m in enumerate(cos.split(sec, dim=-1))], dim=-1).unsqueeze(1)
    sin = torch.cat([m[i % 3] for i, m in enumerate(sin.split(sec, dim=-1))], dim=-1).unsqueeze(1)
    for l in range(cfg["layers"]):
        b = "%slayers.%d." % (p, l)
        h = _rms(x, sd[b + "input_layernorm.weight"], cfg["rms_eps"])
        q = F.linear(h, sd[b + "self_attn.q_proj.weight"].to(dt), sd[b + "self_attn.q_proj.bias"].to(dt))
        k = F.linear(h, sd[b + "self_attn.k_proj.weight"].to(dt), sd[b + "self_attn.k_proj.bias"].to(dt))
        v = F.linear(h, sd[b + "self_attn.v_proj.weight"].to(dt), sd[b + "self_attn.v_proj.bias"].to(dt))
        q = q.view(B, S, heads, hd).transpose(1, 2)
        k = k.view(B, S, kvh, hd).transpose(1, 2)
        v = v.view(B, S, kvh, hd).transpose(1, 2)
        q = q * cos + _rot_half(q) * sin
        k = k * cos + _rot_half(k) * sin
        a = F.scaled_dot_product_attention(q, k, v, is_causal=True, enable_gqa=True)
        x = x + F.linear(a.transpose(1, 2).reshape(B, S, heads * hd), sd[b + "self_attn.o_proj.weight"].to(dt))
        h = _rms(x, sd[b + "post_attention_layernorm.weight"], cfg["rms_eps"])
        g = F.linear(h, sd[b + "mlp.gate_proj.weight"].to(dt))
        u = F.linear(h, sd[b + "mlp.up_proj.weight"].to(dt))
        x = x + F.linear(F.silu(g) * u, sd[b + "mlp.down_proj.weight"].to(dt))
    return _rms(x, sd[p + "norm.weight"], cfg["rms_eps"])


def generate_latents_batched(sd, cfg, input_ids, pixel_values, grid):
    """InternVLAN1ForCausalLM.generate_latents for B equal-length prompts with one image of `grid` each."""
    B, S = input_ids.shape
    dt = pixel_values.dtype
    nq = cfg["n_query"]
    dev = pixel_values.device
    text = sd["model.embed_tokens.weight"][input_ids.to(dev)].to(dt)
    img = vit_forward_batched(sd, cfg, pixel_values, grid, B)
    text[(input_ids == Q.IMAGE_TOKEN_INDEX).to(dev)] = img
    text = torch.cat([text, sd["model.latent_queries"].to(dt).expand(B, -1, -1)], dim=1)
    ids = torch.cat([input_ids, torch.full((B, nq), Q.TRAJ_TOKEN_INDEX)], dim=1)
    pos, _ = Q.rope_index(ids, torch.tensor([list(grid)] * B), cfg["v_merge"])
    return text_forward_batched(sd, cfg, text, pos.to(dev))[:, -nq:, :]


def dual_system_step(sd2, sd1, cfg, input_ids, pixel_values, grid, rgb, depth, x_init, step_noise, K=20):
    """One batched policy step: latents -> System 1 (attention through SDPA) -> trajectories [B * 32, T, 3]."""
    prev = O.ATTENTION
    O.ATTENTION = "sdpa"
    try:
        with torch.no_grad():
            lat = generate_latents_batched(sd2, cfg, input_ids, pixel_values, grid)
            return O.predict_pointgoal_action_async(sd1, lat, rgb, depth, x_init, step_noise, K=K)
    finally:
        O.ATTENTION = prev
