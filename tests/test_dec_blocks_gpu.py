"""Element-wise tests of the fused NavDP decoder attention sublayers (dec_attn_block.cu): the self-attention block
x += W_o MHA_causal(LN1(x) W_qkv^T + b) + b_o and the cross-attention block x += W_o MHA(LN2(x) W_q^T + b_q, K_e, V_e) + b_o.

Every output element is held to a float64 reference that rounds where the kernel rounds (LayerNorm output, q / k / v, P,
O, the output), with the bound built from the helpers of test_hopper_kernels_gpu.py.  The residual stream is a column
slice of a sentinel-filled buffer (row stride > 384) and the sentinels must survive.  A second identical call must
reproduce the first bit for bit, and the first B' environments of a batch must equal a B'-environment call bit for bit
(a tile never spans two environments).  tests/test_dec_blocks_host.py shows on the CPU that the reference and bound
reject a shifted causal mask, a trajectory boundary off by one row and a tile reading its neighbour's K / V.
"""
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_hopper_kernels_gpu import (U32, assert_guard, assert_within, bf16_rounding_risk, elementwise_bound,  # noqa: E402
                                     guarded, random_sign_sum_bound)

pytestmark = pytest.mark.gpu

D, H, HD = 384, 8, 48
SCALE = 1.0 / math.sqrt(HD)


# ------------------------------------------------------------------------------------------ reference
def ln_ref(x, lw, lb, eps):
    """float64 LayerNorm rounded to bf16 as the kernel stores it -> (h, e_h: bound on |kernel h - h|); the fp32 error
    terms are those of test_hopper_kernels_gpu.ff_ref."""
    x64 = x.double()
    mu = x64.mean(-1, keepdim=True)
    xc = x64 - mu
    var = (xc * xc).mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    hn = xc * rstd * lw.double() + lb.double()
    ax = x64.abs()
    q = torch.exp2(torch.floor(torch.log2(ax.clamp_min(2.0 ** -126))) - 7).amin(-1, keepdim=True)
    exact_sum = (ax.sum(-1, keepdim=True) / q) < 2.0 ** 24
    e_mu = torch.where(exact_sum, 2 * U32 * mu.abs(), (D + 8) * U32 * ax.mean(-1, keepdim=True))
    e_rstd = 0.5 * ((D + 16) * U32 * var + e_mu ** 2) / (var + eps) + 4 * U32
    d_h = lw.double().abs() * rstd * (e_mu + xc.abs() * e_rstd) + 4 * U32 * (hn.abs() + lb.double().abs())
    return hn.to(torch.bfloat16).double(), bf16_rounding_risk(hn, d_h)


def proj_ref(h, e_h, w, b):
    """bf16(h W^T + b) as the kernel's projection epilogue rounds it -> (value, bound on the kernel's deviation)."""
    pre = h @ w.double().T + b.double()
    m_pre = h.abs() @ w.double().abs().T + b.double().abs()
    e_pre = (D + 64) * U32 * m_pre + random_sign_sum_bound(e_h, w)
    return pre.to(torch.bfloat16).double(), bf16_rounding_risk(pre, e_pre)


def heads(t, groups):
    """[rows, 384] -> [groups, 8, rows / groups, 48]"""
    return t.view(groups, -1, H, HD).permute(0, 2, 1, 3)


def attn_ref(q, k, v, e_q, e_k, e_v, mask):
    """Softmax attention as the kernel computes it: fp32 logits, P = bf16(exp(s - max)), O = bf16(P V / sum exp).
    q [G, 8, S, 48], k / v [G, 8, Sk, 48] (bf16 values in float64), e_* bounds on the kernel's q / k / v deviations,
    mask [G or 1, 1, S, Sk] bool (True = visible) -> (O [G * S, 384], e_O)."""
    s = (q @ k.transpose(-1, -2)) * SCALE
    e_s = SCALE * (e_q @ k.abs().transpose(-1, -2) + q.abs() @ e_k.transpose(-1, -2) + e_q @ e_k.transpose(-1, -2)
                   + (HD + 64) * U32 * (q.abs() @ k.abs().transpose(-1, -2))) + 8 * U32 * s.abs()
    s = s.masked_fill(~mask, -math.inf)
    m = s.amax(-1, keepdim=True)
    p = torch.exp(s - m)
    # the row maximum and each logit move by at most E: p moves by at most a factor exp(2E), plus exp2f's few ulp
    E = e_s.masked_fill(~mask, 0.0).amax(-1, keepdim=True)
    rel = torch.expm1(2 * E) + 16 * U32
    P = p.to(torch.bfloat16).double()
    e_P = bf16_rounding_risk(p, p * rel)
    l = p.sum(-1, keepdim=True)
    e_l = (p * rel).sum(-1, keepdim=True) + 64 * U32 * l
    num = P @ v
    e_num = e_P @ v.abs() + P @ e_v + 128 * U32 * (P @ v.abs())
    o = num / l
    e_o = e_num / l + o.abs() * e_l / l + 4 * U32 * o.abs()
    G, _, S, _ = q.shape
    flat = lambda t: t.permute(0, 2, 1, 3).reshape(G * S, H * HD)
    o, e_o = flat(o), flat(e_o)
    return o.to(torch.bfloat16).double(), bf16_rounding_risk(o, e_o)


def out_ref(x, O, e_O, wo, bo):
    x64 = x.double()
    out = x64 + O @ wo.double().T + bo.double()
    mag = x64.abs() + O.abs() @ wo.double().abs().T + bo.double().abs()
    return out, elementwise_bound(out, mag, D, extra=random_sign_sum_bound(e_O, wo))


def sa_ref(x, p, B, Ns, T, causal, eps=1e-5, key_shift=0, row_shift=0):
    """Self-attention block -> (out, bound).  key_shift / row_shift model wrong kernels (host test): a causal mask that
    lets row i see key i + key_shift, and trajectory boundaries moved by row_shift rows."""
    h, e_h = ln_ref(x, p["ln_w"], p["ln_b"], eps)
    qkv, e_qkv = proj_ref(h, e_h, p["w_in"], p["b_in"])
    G = B if row_shift else B * Ns     # attention groups: trajectories, or whole environments when boundaries move
    S = Ns * T if row_shift else T
    r = torch.arange(S, device=x.device)
    traj = (r + row_shift).div(T, rounding_mode="floor")
    mask = traj[:, None] == traj[None, :]
    if causal:
        mask &= r[None, :] <= r[:, None] + key_shift
    parts = [heads(t[:, i * D:(i + 1) * D], G) for t in (qkv, e_qkv) for i in range(3)]
    O, e_O = attn_ref(parts[0], parts[1], parts[2], parts[3], parts[4], parts[5], mask[None, None])
    return out_ref(x, O, e_O, p["w_o"], p["b_o"])


def ca_ref(x, p, kv, mtok, B, Ns, T, eps=1e-5, env_shift=0):
    """Cross-attention block -> (out, bound).  kv [B * mtok, >= 768] (K | V).  env_shift models a wrong kernel
    (host test): environment 0 reads the K / V of environment env_shift."""
    h, e_h = ln_ref(x, p["ln_w"], p["ln_b"], eps)
    q, e_q = proj_ref(h, e_h, p["w_in"], p["b_in"])
    kv64 = kv[:, :2 * D].double().view(B, mtok, 2 * D)
    if env_shift:
        kv64 = kv64.clone()
        kv64[0] = kv64[env_shift % B]
    k = kv64[..., :D].reshape(B, mtok, H, HD).permute(0, 2, 1, 3)
    v = kv64[..., D:].reshape(B, mtok, H, HD).permute(0, 2, 1, 3)
    z = torch.zeros_like(k)
    mask = torch.ones(1, 1, 1, mtok, dtype=torch.bool, device=x.device)
    O, e_O = attn_ref(heads(q, B), k, v, heads(e_q, B), z, z, mask)
    return out_ref(x, O, e_O, p["w_o"], p["b_o"])


def make_params(self_attn, seed, device="cpu"):
    """Weights like a trained layer's in scale; W_q is 3x larger so that the logits spread over ~+-10 and a wrong mask
    moves the output far more than the bound allows."""
    gen = torch.Generator().manual_seed(seed)
    n_in = 3 * D if self_attn else D
    w_in = torch.randn(n_in, D, generator=gen) / math.sqrt(D)
    w_in[:D] *= 3.0
    p = dict(w_in=w_in.bfloat16(), b_in=torch.randn(n_in, generator=gen) * 0.1,
             w_o=(torch.randn(D, D, generator=gen) / math.sqrt(D)).bfloat16(), b_o=torch.randn(D, generator=gen) * 0.1,
             ln_w=1 + 0.1 * torch.randn(D, generator=gen), ln_b=0.1 * torch.randn(D, generator=gen))
    return {k: v.to(device) for k, v in p.items()}


def make_x(R, seed, device="cpu"):
    """Rows of three kinds (as the FF-block test): offset 100 + N(0, 1), N(0.3, 1.5^2) and N(0, 2^-18)."""
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(R, D, generator=gen)
    kind = torch.arange(R) % 3
    x[kind == 0] += 100.0
    x[kind == 1] = x[kind == 1] * 1.5 + 0.3
    x[kind == 2] *= 2.0 ** -9
    return x.bfloat16().to(device)


def make_kv(B, mtok, seed, device="cpu"):
    """K / V of every environment as a column slice of a wider buffer, as the decoder's stacked per-layer K / V are."""
    gen = torch.Generator().manual_seed(seed)
    buf = (torch.randn(B * mtok, 4 * D, generator=gen) * 1.5).bfloat16().to(device)
    return buf[:, 2 * D:]


# ------------------------------------------------------------------------------------------ GPU runs
@pytest.fixture(scope="module")
def L():
    from internnav_b200 import _lib
    _lib.lib()
    return _lib


def _run(L, self_attn, x, p, B, Ns, T, causal=True, kv=None, mtok=0):
    """The block on a copy of x inside a guarded buffer (ldx = 384 + 40); checks the sentinels; returns the result."""
    xbuf, xv = guarded(x.shape[0], D, torch.bfloat16, "cuda", left=16, right=24)
    xv.copy_(x)
    if self_attn:
        L.dec_sa_block(xv, p["ln_w"], p["ln_b"], p["w_in"], p["b_in"], p["w_o"], p["b_o"], B, Ns, T, causal=causal)
    else:
        L.dec_ca_block(xv, p["ln_w"], p["ln_b"], p["w_in"], p["b_in"], p["w_o"], p["b_o"], kv, mtok, B, Ns, T)
    torch.cuda.synchronize()
    assert_guard(xbuf, xv, "dec block x")
    return xv.clone()


def _check(L, self_attn, B, Ns, T, causal=True, mtok=0, seed=0):
    p = make_params(self_attn, seed, "cuda")
    R = B * Ns * T
    x = make_x(R, seed + 1, "cuda")
    kv = make_kv(B, mtok, seed + 2, "cuda") if not self_attn else None
    out = _run(L, self_attn, x, p, B, Ns, T, causal, kv, mtok)
    if self_attn:
        ref, bound = sa_ref(x, p, B, Ns, T, causal)
    else:
        ref, bound = ca_ref(x, p, kv, mtok, B, Ns, T)
    what = "%s B=%d Ns=%d T=%d%s" % ("sa" if self_attn else "ca", B, Ns, T, "" if self_attn else " mtok=%d" % mtok)
    assert_within(out, ref, bound, what)
    again = _run(L, self_attn, x, p, B, Ns, T, causal, kv, mtok)
    assert torch.equal(out.view(torch.int16), again.view(torch.int16)), what + ": second call differs"
    if B > 1:   # the first environments alone give the same rows, bit for bit
        Bp = max(1, B // 2)
        part = _run(L, self_attn, x[:Bp * Ns * T], p, Bp, Ns, T, causal, kv[:Bp * mtok] if kv is not None else None, mtok)
        assert torch.equal(part.view(torch.int16), out[:Bp * Ns * T].view(torch.int16)), what + ": batch prefix differs"


SA_CASES = [(2, 5, 8), (3, 5, 17), (2, 5, 24), (2, 32, 32), (1, 1, 32), (3, 32, 8), (1, 529, 32)]   # last: 2 x 132 + 1 tiles


@pytest.mark.parametrize("B,Ns,T", SA_CASES)
def test_sa_block(L, B, Ns, T):
    _check(L, True, B, Ns, T, causal=True, seed=B * 1000 + Ns * 40 + T)


@pytest.mark.parametrize("T", [17, 32])
def test_sa_block_not_causal(L, T):
    _check(L, True, 2, 5, T, causal=False, seed=7 + T)


@pytest.mark.parametrize("mtok", [1, 34, 64])
@pytest.mark.parametrize("B,Ns,T", [(2, 5, 8), (3, 5, 17), (2, 5, 24), (2, 32, 32), (1, 1, 32), (3, 1, 24), (1, 529, 32)])
def test_ca_block(L, B, Ns, T, mtok):
    _check(L, False, B, Ns, T, mtok=mtok, seed=B * 1000 + Ns * 40 + T + mtok)
