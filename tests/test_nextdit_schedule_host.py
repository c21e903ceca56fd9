"""The NextDiT launch schedule (internnav_b200/nextdit.py: weight packing, hoisted conditioning, group-indexed modulation,
cross-attention K / V sharing, guidance batch, Euler update) executed on the CPU with every library op replaced by a plain
PyTorch stand-in that enforces the kernels' operand contracts -- against the oracle and the reference-run fixture.  The same
idea as tests/test_train_s1_host.py: the schedule is host logic and must be testable without a GPU; the kernels
themselves are tested against the same stand-ins' arithmetic on the H100 (tests/test_nextdit_gpu.py, test_ops_gpu.py)."""
import math
import os
import types

import numpy as np
import torch
import torch.nn.functional as F

from internnav_b200 import nextdit as N
from internnav_b200.manifest import random_nextdit_state_dict

GOLD = os.path.join(os.path.dirname(__file__), "golden", "nextdit_reference.npz")
BF = torch.bfloat16


def _rows(t):
    assert t.dim() == 2 and t.stride(1) == 1, ("kernel operands are row-major views with unit inner stride", t.shape, t.stride())
    return t.float()


class FakeLib:
    """fp32 arithmetic on the bf16 operands, bf16 results: what the kernels compute, up to summation order."""
    ACT_NONE, ACT_GELU, ACT_RELU, ACT_SWIGLU, ACT_GELU_TANH, ACT_SILU = 0, 1, 2, 3, 4, 5
    calls = {}

    @classmethod
    def _c(cls, k):
        cls.calls[k] = cls.calls.get(k, 0) + 1

    @classmethod
    def gemm(cls, a, w, bias=None, gamma=None, residual=None, act=0, out_fp32=False, out=None):
        cls._c("gemm")
        assert a.dtype == BF and w.dtype == BF and a.shape[1] == w.shape[1] and a.shape[1] % 8 == 0 and w.shape[0] % 8 == 0
        y = _rows(a) @ _rows(w).t()
        if bias is not None:
            assert bias.dtype == torch.float32 and bias.is_contiguous()
            y = y + bias
        if act == cls.ACT_SWIGLU:
            y = F.silu(y[:, 0::2]) * y[:, 1::2]
        elif act:
            y = {1: F.gelu, 2: F.relu, 4: lambda t: F.gelu(t, approximate="tanh"), 5: F.silu}[act](y)
        if gamma is not None:
            y = y * gamma
        if residual is not None:
            y = y + _rows(residual)
        return y if out_fp32 else y.to(BF)

    @classmethod
    def layernorm(cls, x, w, b=None, eps=1e-5, rms=False, out=None):
        cls._c("layernorm")
        assert x.dtype == BF and w.dtype == torch.float32 and not rms
        y = F.layer_norm(_rows(x), (x.shape[1],), w, b, eps).to(BF)
        if out is not None:
            assert out.shape == x.shape and out.stride(1) == 1
            out.copy_(y)
            return out
        return y

    @classmethod
    def attention(cls, q, k, v, heads_q, heads_kv, head_dim, batch, seq_q, seq_k, kv_div=1, causal=False, scale=None, **kw):
        cls._c("attention")
        assert heads_q == heads_kv and not causal and batch % kv_div == 0
        D = heads_q * head_dim
        assert q.shape == (batch * seq_q, D) and k.shape == (batch // kv_div * seq_k, D) and v.shape == k.shape
        qh = _rows(q).view(batch, seq_q, heads_q, head_dim).transpose(1, 2)
        kh = _rows(k).view(batch // kv_div, seq_k, heads_q, head_dim).transpose(1, 2).repeat_interleave(kv_div, dim=0)
        vh = _rows(v).view(batch // kv_div, seq_k, heads_q, head_dim).transpose(1, 2).repeat_interleave(kv_div, dim=0)
        s = qh @ kh.transpose(-1, -2) * (head_dim ** -0.5 if scale is None else scale)
        return (s.softmax(-1) @ vh).transpose(1, 2).reshape(batch * seq_q, D).to(BF)

    @classmethod
    def mod_norm(cls, x, w, mod, rows_per_group, eps, mode, residual=None, out=None):
        cls._c("mod_norm")
        xf = _rows(x)
        if mode == 1:
            y = F.layer_norm(xf, (x.shape[1],), None, None, eps)
        else:
            y = xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps)
        if w is not None:
            y = y * w
        if mod is not None:
            assert mod.dtype == BF and mod.stride(1) == 1 and mod.shape[0] * rows_per_group == x.shape[0]
            m = mod.float().repeat_interleave(rows_per_group, dim=0)
            y = y * (torch.tanh(m) if mode == 2 else 1 + m)
        if mode == 2:
            y = y + _rows(residual)
        return y.to(BF)

    @classmethod
    def add(cls, a, b, out=None):
        cls._c("add")
        return (a.float() + b.float()).to(BF)

    @classmethod
    def action_embed(cls, lat, w, b, pos, out=None):
        cls._c("action_embed")
        assert lat.dtype == torch.float32 and lat.is_contiguous()
        rows = lat.reshape(-1, 3)
        y = ((rows @ w.t() + b).to(BF).float() + pos.repeat(rows.shape[0] // pos.shape[0], 1)).to(BF)
        if out is not None:
            out.copy_(y)
            return out
        return y

    @classmethod
    def cfg_euler(cls, pred, n, cfg, scale, dt, lat):
        cls._c("cfg_euler")
        p = pred[:, :3].float()
        if cfg:
            u, c = p[:n], p[n:]
            p = (u + (scale * (c - u).to(BF).float()).to(BF).float()).to(BF).float()
        flat = lat.view(-1, 3)
        flat.copy_((flat + (dt * p).to(BF).float()).to(BF).float())
        return lat


class FakeBwd:
    @staticmethod
    def patchify_depth(frames, ldk=200):
        n = frames.shape[0]
        p = frames.reshape(n, 16, 14, 16, 14).permute(0, 1, 3, 2, 4).reshape(n * 256, 196)
        return F.pad(p, (0, ldk - 196)).to(BF)


def _system(monkeypatch, seed):
    monkeypatch.setattr(N, "_lib", FakeLib)
    monkeypatch.setattr(N, "_bwd", FakeBwd)
    FakeLib.calls = {}
    m = object.__new__(N.NextDiTSystem1)
    m.device, m.num_inference_steps, m.w = torch.device("cpu"), 10, None
    return m.load_state_dict(random_nextdit_state_dict(seed))


def _rel(a, b):
    a, b = torch.as_tensor(a).float(), torch.as_tensor(b).float()
    return float((a - b).norm() / (b.norm() + 1e-12))


def test_schedule_reproduces_the_reference_run(monkeypatch):
    from oracle.gen_golden_nextdit import make_inputs
    g = np.load(GOLD)
    m = _system(monkeypatch, int(g["seed"]))
    inp = make_inputs(int(g["seed"]), int(g["batch"]), int(g["ns"]))
    cond = m.condition_tokens(inp["traj_latents"], inp["images_dp"])
    assert cond.shape == (1, 36, 768) and _rel(cond, g["condition_tokens"]) < 2e-2
    for scale, key, exact in ((1.0, "traj_scale_1", False), (1.0, "traj_scale_1", True), (2.5, "traj_scale_2p5", False)):
        out = m.generate_traj(inp["traj_latents"], inp["images_dp"], guidance_scale=scale, num_sample_trajs=int(g["ns"]),
                              x_init=inp["x_init"], exact_cfg=exact, graph=False)
        assert out.shape == (3, 32, 3) and _rel(out, g[key]) < 3e-2, (scale, exact, _rel(out, g[key]))
    # what was hoisted out of the loop really ran once per call: per sampler call 12 x 10 block evaluations with 5 GEMMs each
    assert FakeLib.calls["cfg_euler"] == 30 and FakeLib.calls["attention"] >= 3 * (12 * 10 * 2)


def test_batch_of_environments_equals_single_calls(monkeypatch):
    m = _system(monkeypatch, 7)
    gen = torch.Generator().manual_seed(5)
    B, Ns = 2, 2
    lat = torch.randn(B, 4, 3584, generator=gen)
    img = torch.rand(B, 2, 224, 224, 3, generator=gen)
    x0 = torch.randn(B * Ns, 32, 3, generator=gen).to(BF)
    full = m.generate_traj(lat, img, guidance_scale=2.0, num_sample_trajs=Ns, x_init=x0, graph=False, num_inference_steps=3)
    for b in range(B):
        one = m.generate_traj(lat[b:b + 1], img[b:b + 1], guidance_scale=2.0, num_sample_trajs=Ns, x_init=x0[b * Ns:(b + 1) * Ns],
                              graph=False, num_inference_steps=3)
        assert _rel(one, full[b * Ns:(b + 1) * Ns]) < 2e-2     # group indexing / kv_div keep the environments apart
