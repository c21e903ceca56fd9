"""Kernel-level parity (through the C ABI) against fp32 PyTorch references of the same op."""
import math

import numpy as np
import os

import pytest
import torch

pytestmark = pytest.mark.gpu


def _rel(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / (b.norm() + 1e-12)).item()


@pytest.fixture(scope="module")
def L():
    from internnav_b200 import _lib
    _lib.lib()
    return _lib


# (M, N, K): tails in every dimension, K not a multiple of 64, tiny M, all three tile widths
GEMM_SHAPES = [(128, 128, 64), (128, 256, 384), (300, 1152, 384), (2048, 384, 1536), (1, 384, 384), (272, 12288, 384),
               (1000, 64, 128), (257 * 4, 384, 592), (4096, 1536, 384), (333, 896, 3584), (64, 448, 896),
               (20000, 1152, 384), (1024, 3584, 3584)]


@pytest.mark.parametrize("M,N,K", GEMM_SHAPES)
def test_gemm_plain(L, M, N, K):
    torch.manual_seed(M + N + K)
    a = torch.randn(M, K, device="cuda").bfloat16()
    w = (torch.randn(N, K, device="cuda") / math.sqrt(K)).bfloat16()
    out = L.gemm(a, w)
    ref = a.float() @ w.float().T
    assert _rel(out, ref) < 6e-3, _rel(out, ref)


@pytest.mark.parametrize("act", [0, 1, 2])
def test_gemm_epilogue(L, act):
    torch.manual_seed(act)
    M, N, K = 777, 384, 1536
    a = torch.randn(M, K, device="cuda").bfloat16()
    w = (torch.randn(N, K, device="cuda") / math.sqrt(K)).bfloat16()
    bias = torch.randn(N, device="cuda")
    gamma = torch.randn(N, device="cuda")
    res = torch.randn(M, N, device="cuda").bfloat16()
    out = L.gemm(a, w, bias=bias, gamma=gamma, residual=res, act=act)
    ref = a.float() @ w.float().T + bias
    if act == 1:
        ref = torch.nn.functional.gelu(ref)
    elif act == 2:
        ref = torch.relu(ref)
    ref = ref * gamma + res.float()
    assert _rel(out, ref) < 6e-3
    # in-place residual (out aliases residual) as the executors use it
    res2 = res.clone()
    L.gemm(a, w, bias=bias, gamma=gamma, residual=res2, act=act, out=res2)
    assert _rel(res2, ref) < 6e-3
    # fp32 output
    out32 = L.gemm(a, w, bias=bias, act=act, out_fp32=True)
    ref32 = a.float() @ w.float().T + bias
    if act == 1:
        ref32 = torch.nn.functional.gelu(ref32)
    elif act == 2:
        ref32 = torch.relu(ref32)
    assert _rel(out32, ref32) < 1e-5 + 2e-3 * 0  or _rel(out32, ref32) < 2e-3


def test_gemm_swiglu(L):
    torch.manual_seed(3)
    M, F, K = 500, 1728, 1280
    a = torch.randn(M, K, device="cuda").bfloat16()
    wg = (torch.randn(F, K, device="cuda") / math.sqrt(K)).bfloat16()
    wu = (torch.randn(F, K, device="cuda") / math.sqrt(K)).bfloat16()
    bg, bu = torch.randn(F, device="cuda"), torch.randn(F, device="cuda")
    w = torch.stack([wg, wu], 1).reshape(2 * F, K).contiguous()
    b = torch.stack([bg, bu], 1).reshape(2 * F).contiguous()
    out = L.gemm(a, w, bias=b, act=3)
    g = a.float() @ wg.float().T + bg
    u = a.float() @ wu.float().T + bu
    ref = torch.nn.functional.silu(g) * u
    assert out.shape == (M, F)
    assert _rel(out, ref) < 6e-3


def test_gemm_strided(L):
    torch.manual_seed(4)
    M, N, K = 64, 768, 384
    big = torch.randn(M, 34 * K, device="cuda").bfloat16()
    a = big[:, :K]  # row stride 34*K, like the time-token refresh in the denoiser
    w = (torch.randn(N, K, device="cuda") / math.sqrt(K)).bfloat16()
    outbig = torch.zeros(M, 34 * N, device="cuda", dtype=torch.bfloat16)
    out = outbig[:, :N]
    L.gemm(a, w, out=out)
    assert _rel(out, a.float() @ w.float().T) < 6e-3
    assert outbig[:, N:].abs().max().item() == 0


@pytest.mark.parametrize("rows,D,rms", [(1000, 384, False), (37, 1280, True), (515, 3584, True), (9, 5120, False),
                                        (4096, 384, False)])
def test_layernorm(L, rows, D, rms):
    torch.manual_seed(rows)
    x = (torch.randn(rows, D, device="cuda") * 3 + 1).bfloat16()
    w = torch.randn(D, device="cuda")
    b = None if rms else torch.randn(D, device="cuda")
    y = L.layernorm(x, w, b, eps=1e-6, rms=rms)
    xf = x.float()
    if rms:
        ref = xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-6) * w
    else:
        ref = torch.nn.functional.layer_norm(xf, (D,), w, b, 1e-6)
    assert _rel(y, ref) < 4e-3


def _ref_attn(q, k, v, causal, scale):
    # q [B,Hq,Sq,d], k/v [B,Hk,Sk,d] fp32
    B, Hq, Sq, d = q.shape
    Hk, Sk = k.shape[1], k.shape[2]
    k = k.repeat_interleave(Hq // Hk, 1)
    v = v.repeat_interleave(Hq // Hk, 1)
    s = (q @ k.transpose(-1, -2)) * scale
    if causal:
        i = torch.arange(Sq, device=q.device)[:, None]
        j = torch.arange(Sk, device=q.device)[None, :]
        s = s.masked_fill(j > i + (Sk - Sq), float("-inf"))
    return s.softmax(-1) @ v


ATTN_CASES = [
    # B, Hq, Hk, hd, Sq, Sk, causal
    (5, 6, 6, 64, 257, 257, False),    # DINOv2
    (64, 8, 8, 48, 8, 8, True),        # denoiser self-attn T=8
    (16, 8, 8, 48, 32, 32, True),      # denoiser self-attn T=32
    (3, 8, 8, 48, 32, 1024, False),    # Q-former cross
    (7, 8, 8, 48, 1, 4, False),        # goal compressor
    (2, 16, 16, 80, 64, 64, False),    # Qwen ViT window
    (2, 16, 16, 80, 784, 784, False),  # Qwen ViT full
    (3, 28, 4, 128, 304, 304, True),   # LLM prefill GQA
    (1, 28, 4, 128, 200, 456, True),   # causal with seq_k > seq_q (bottom-right aligned)
]


@pytest.mark.parametrize("B,Hq,Hk,hd,Sq,Sk,causal", ATTN_CASES)
def test_attention_fixed(L, B, Hq, Hk, hd, Sq, Sk, causal):
    torch.manual_seed(B * Sq + hd)
    q = torch.randn(B * Sq, Hq * hd, device="cuda").bfloat16()
    k = torch.randn(B * Sk, Hk * hd, device="cuda").bfloat16()
    v = torch.randn(B * Sk, Hk * hd, device="cuda").bfloat16()
    o = L.attention(q, k, v, Hq, Hk, hd, B, Sq, Sk, causal=causal)
    ref = _ref_attn(q.float().view(B, Sq, Hq, hd).transpose(1, 2), k.float().view(B, Sk, Hk, hd).transpose(1, 2),
                    v.float().view(B, Sk, Hk, hd).transpose(1, 2), causal, hd ** -0.5)
    ref = ref.transpose(1, 2).reshape(B * Sq, Hq * hd)
    assert _rel(o, ref) < 8e-3, _rel(o, ref)


def test_attention_packed_qkv_and_shared_kv(L):
    """q/k/v as column slices of one packed buffer; 32 samples share one environment's memory (kv_div)."""
    torch.manual_seed(0)
    B, Ns, T, M, H, hd = 3, 32, 8, 34, 8, 48
    D = H * hd
    qkv = torch.randn(B * Ns * T, 3 * D, device="cuda").bfloat16()
    o = L.attention(qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:], H, H, hd, B * Ns, T, T, causal=True)
    q4 = qkv.float().view(B * Ns, T, 3, H, hd)
    ref = _ref_attn(q4[:, :, 0].transpose(1, 2), q4[:, :, 1].transpose(1, 2), q4[:, :, 2].transpose(1, 2), True,
                    hd ** -0.5).transpose(1, 2).reshape(B * Ns * T, D)
    assert _rel(o, ref) < 8e-3
    # cross attention to per-environment memory with a wide stride (layer slice of the stacked K/V buffer)
    ckv = torch.randn(B * M, 16 * 2 * D, device="cuda").bfloat16()
    l = 5
    kk, vv = ckv[:, l * 2 * D:l * 2 * D + D], ckv[:, l * 2 * D + D:(l + 1) * 2 * D]
    q = torch.randn(B * Ns * T, D, device="cuda").bfloat16()
    o = L.attention(q, kk, vv, H, H, hd, B * Ns, T, M, kv_div=Ns)
    kf = kk.float().view(B, M, H, hd).transpose(1, 2).repeat_interleave(Ns, 0)
    vf = vv.float().view(B, M, H, hd).transpose(1, 2).repeat_interleave(Ns, 0)
    ref = _ref_attn(q.float().view(B * Ns, T, H, hd).transpose(1, 2), kf, vf, False, hd ** -0.5)
    ref = ref.transpose(1, 2).reshape(B * Ns * T, D)
    assert _rel(o, ref) < 8e-3


def test_attention_varlen(L):
    torch.manual_seed(1)
    H, hd = 16, 80
    lens = [64, 64, 48, 784, 1, 130]
    cu = torch.tensor([0] + list(torch.tensor(lens).cumsum(0)), device="cuda", dtype=torch.int32)
    tot = sum(lens)
    q = torch.randn(tot, H * hd, device="cuda").bfloat16()
    k = torch.randn(tot, H * hd, device="cuda").bfloat16()
    v = torch.randn(tot, H * hd, device="cuda").bfloat16()
    for causal in (False, True):
        o = L.attention(q, k, v, H, H, hd, len(lens), 0, 0, cu_q=cu, cu_k=cu, max_seq_q=max(lens), causal=causal)
        s = 0
        for n in lens:
            sl = slice(s, s + n)
            ref = _ref_attn(q[sl].float().view(1, n, H, hd).transpose(1, 2), k[sl].float().view(1, n, H, hd).transpose(1, 2),
                            v[sl].float().view(1, n, H, hd).transpose(1, 2), causal, hd ** -0.5)
            assert _rel(o[sl], ref.transpose(1, 2).reshape(n, H * hd)) < 8e-3
            s += n


@pytest.mark.parametrize("M,seed", [(128, 1), (1000, 1), (256, 2), (1000, 2), (65536 // 8, 2), (300, 2), (65536, 2)])
def test_ff_block_vs_fp32_and_unfused(L, M, seed):
    """FF block of the NavDP decoder layer in one kernel (ff_block.cu): LayerNorm + linear1 + GELU + linear2 + residual,
    residual stream in tensor memory; against fp32 PyTorch on the same bf16 inputs."""
    torch.manual_seed(M + seed)
    x = (torch.randn(M, 384, device="cuda") * 1.5 + 0.3).bfloat16()
    w1 = (torch.randn(1536, 384, device="cuda") / math.sqrt(384)).bfloat16()
    w2 = (torch.randn(384, 1536, device="cuda") / math.sqrt(1536)).bfloat16()
    b1, b2 = torch.randn(1536, device="cuda") * 0.1, torch.randn(384, device="cuda") * 0.1
    lw, lb = 1 + 0.1 * torch.randn(384, device="cuda"), 0.1 * torch.randn(384, device="cuda")
    h = torch.nn.functional.layer_norm(x.float(), (384,), lw, lb, 1e-5).bfloat16().float()   # the kernel's operand is bf16
    ref = x.float() + torch.nn.functional.gelu(h @ w1.float().T + b1) @ w2.float().T + b2
    out = L.ff_block(x, lw, lb, w1, b1, w2, b2)
    torch.cuda.synchronize()
    assert _rel(out, ref) < 6e-3, _rel(out, ref)
    # in place on the residual stream, as the decoder uses it; twice in a row (persistent state must not leak)
    r2 = x.clone()
    L.ff_block(r2, lw, lb, w1, b1, w2, b2, out=r2)
    assert torch.equal(r2, out)
    # the unfused kernels of the library compute the same block (LayerNorm -> GEMM+GELU -> GEMM+residual)
    hk = L.layernorm(x, lw, lb, 1e-5)
    hid = L.gemm(hk, w1, bias=b1, act=L.ACT_GELU)
    un = L.gemm(hid, w2, bias=b2, residual=x)
    assert _rel(out, un) < 6e-3, _rel(out, un)

@pytest.mark.parametrize("lens,causal", [([304] * 4, True), ([304, 300, 129, 128, 1, 257, 320, 64, 17], True),
                                         ([320, 200, 96], False), ([304] * 64, True)])
def test_attention_tcgen05_hd128(L, lens, causal):
    """Decoder-prefill attention on wgmma (attention_wgmma.cu): var-len GQA 28 / 4, head_dim 128, packed q|k|v rows with the
    decoder's row stride; against fp32 PyTorch per sequence and against the mma.sync kernel it replaces."""
    torch.manual_seed(len(lens) + sum(lens))
    Hq, Hkv, hd = 28, 4, 128
    T = sum(lens)
    qkv = torch.randn(T, (Hq + 2 * Hkv) * hd, device="cuda").bfloat16()
    q, k, v = qkv[:, :Hq * hd], qkv[:, Hq * hd:(Hq + Hkv) * hd], qkv[:, (Hq + Hkv) * hd:]
    cu = torch.tensor([0] + list(np.cumsum(lens)), dtype=torch.int32, device="cuda")
    o, used = L.attention_varlen(q, k, v, Hq, Hkv, hd, cu, max(lens), causal=causal)
    assert used, "the wgmma kernel should take this shape"
    old = L.attention(q, k, v, Hq, Hkv, hd, len(lens), 0, 0, cu_q=cu, cu_k=cu, max_seq_q=max(lens), causal=causal)
    s = 0
    worst = 0.0
    for n in lens[:12]:
        sl = slice(s, s + n)
        qh = q[sl].float().view(n, Hq, hd).transpose(0, 1)
        kh = k[sl].float().view(n, Hkv, hd).transpose(0, 1).repeat_interleave(Hq // Hkv, dim=0)
        vh = v[sl].float().view(n, Hkv, hd).transpose(0, 1).repeat_interleave(Hq // Hkv, dim=0)
        sc = qh @ kh.transpose(-1, -2) * hd ** -0.5
        if causal:
            sc = sc.masked_fill(torch.triu(torch.ones(n, n, dtype=torch.bool, device="cuda"), 1), float("-inf"))
        ref = (sc.softmax(-1) @ vh).transpose(0, 1).reshape(n, Hq * hd)
        worst = max(worst, _rel(o[sl], ref))
        s += n
    assert worst < 8e-3, worst
    assert _rel(o, old) < 8e-3
