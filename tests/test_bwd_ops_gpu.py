"""Backward primitives (csrc/bwd_kernels.cu) against PyTorch autograd / torch.optim on the GPU."""
import math
import os

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def _rel(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / (b.norm() + 1e-12))


def test_transpose_and_colsum():
    from internnav_b200 import _bwd as K
    torch.manual_seed(0)
    for rows, cols in [(257, 384), (2048, 1536), (5, 48), (1000, 3)]:
        x = torch.randn(rows, cols, device="cuda").bfloat16()
        t = K.transpose(x)
        assert t.shape == (cols, (rows + 7) // 8 * 8)
        assert torch.equal(t[:, :rows], x.t()) and float(t[:, rows:].abs().max() if t.shape[1] > rows else 0) == 0
        y = torch.randn(rows, cols, device="cuda").bfloat16()
        assert _rel(K.colsum(x), x.float().sum(0)) < 1e-5
        assert _rel(K.colsum(x, y), (x.float() * y.float()).sum(0)) < 1e-5


@pytest.mark.parametrize("rows,D,rms", [(300, 384, False), (4100, 384, False), (64, 3584, True), (257, 384, False)])
def test_norm_bwd(rows, D, rms):
    from internnav_b200 import _bwd as K
    torch.manual_seed(rows)
    x = torch.randn(rows, D, device="cuda").bfloat16()
    w = (1 + 0.1 * torch.randn(D, device="cuda"))
    b = 0.1 * torch.randn(D, device="cuda")
    dy = torch.randn(rows, D, device="cuda").bfloat16()
    rg = torch.randn(rows, D, device="cuda").bfloat16()
    eps = 1e-6 if rms else 1e-5
    xf = x.float().requires_grad_(True)
    wf, bf = w.clone().requires_grad_(True), b.clone().requires_grad_(True)
    if rms:
        y = wf * (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps))
    else:
        y = torch.nn.functional.layer_norm(xf, (D,), wf, bf, eps)
    y.backward(dy.float())
    dx, dw, db = K.norm_bwd(dy, x, w, eps, rms=rms, residual_grad=rg)
    assert _rel(dx, xf.grad + rg.float()) < 6e-3
    assert _rel(dw, wf.grad) < 2e-3
    if not rms:
        assert _rel(db, bf.grad) < 2e-3


def test_activation_backward():
    from internnav_b200 import _bwd as K
    torch.manual_seed(1)
    pre = (2 * torch.randn(1000, 1536, device="cuda")).bfloat16()
    dy = torch.randn(1000, 1536, device="cuda").bfloat16()
    for act, fn in [(1, torch.nn.functional.gelu), (2, torch.relu)]:
        p = pre.float().requires_grad_(True)
        fn(p).backward(dy.float())
        assert _rel(K.act_bwd(pre, dy, act), p.grad) < 5e-3
    g = torch.randn(64, 2 * 512, device="cuda").bfloat16()     # interleaved (gate, up)
    da = torch.randn(64, 512, device="cuda").bfloat16()
    p = g.float().requires_grad_(True)
    (torch.nn.functional.silu(p[:, 0::2]) * p[:, 1::2]).backward(da.float())
    assert _rel(K.swiglu_bwd(g, da), p.grad) < 5e-3


def test_rope_transposed_is_the_adjoint():
    from internnav_b200 import _bwd as K
    torch.manual_seed(2)
    rows, heads, hd = 37, 5, 128
    ang = torch.rand(rows, hd // 2, device="cuda") * 6.28
    cs = torch.stack((ang.cos(), ang.sin()), dim=-1).contiguous()
    x = torch.randn(rows, heads * hd, device="cuda")
    y = torch.randn(rows, heads * hd, device="cuda")

    def rope(t):
        t = t.view(rows, heads, hd)
        c, s = torch.cat((ang.cos(), ang.cos()), -1)[:, None], torch.cat((ang.sin(), ang.sin()), -1)[:, None]
        rot = torch.cat((-t[..., hd // 2:], t[..., : hd // 2]), dim=-1)
        return (t * c + rot * s).reshape(rows, heads * hd)
    yt = K.rope_transposed(y.bfloat16().clone(), cs, heads, hd).float()
    lhs, rhs = (rope(x) * y.bfloat16().float()).sum(), (x * yt).sum()     # <R x, y> = <x, R^T y>
    assert abs(float(lhs - rhs)) < 2e-2 * float(x.norm() * y.norm()) / math.sqrt(rows)


@pytest.mark.parametrize("B,Sq,Sk,Hq,Hkv,hd,causal", [(6, 32, 32, 8, 8, 48, True), (6, 32, 34, 8, 8, 48, False),
                                                      (3, 257, 257, 6, 6, 64, False), (2, 32, 1024, 8, 8, 48, False),
                                                      (2, 4, 300, 28, 4, 128, True), (1, 1, 4, 8, 8, 48, False),
                                                      (2, 40, 72, 6, 6, 64, True), (5, 100, 100, 6, 6, 64, True)])
def test_attention_bwd(B, Sq, Sk, Hq, Hkv, hd, causal):
    """Fixed-length MHA with head_dim 48 / 64 whose four operand tiles fit the shared memory of an SM runs the tensor-core
    kernel (attention_bwd_mma.cu); GQA, head_dim 128 and the 1024-key case run the scalar kernel (bwd_kernels.cu)."""
    from internnav_b200 import _bwd as K, _lib as L
    torch.manual_seed(B * Sq + Sk)
    q = torch.randn(B * Sq, Hq * hd, device="cuda").bfloat16()
    k = torch.randn(B * Sk, Hkv * hd, device="cuda").bfloat16()
    v = torch.randn(B * Sk, Hkv * hd, device="cuda").bfloat16()
    do = torch.randn(B * Sq, Hq * hd, device="cuda").bfloat16()
    qf, kf, vf = (t.float().requires_grad_(True) for t in (q, k, v))
    qh = qf.view(B, Sq, Hq, hd).transpose(1, 2)
    kh = kf.view(B, Sk, Hkv, hd).transpose(1, 2).repeat_interleave(Hq // Hkv, dim=1)
    vh = vf.view(B, Sk, Hkv, hd).transpose(1, 2).repeat_interleave(Hq // Hkv, dim=1)
    s = qh @ kh.transpose(-1, -2) * hd ** -0.5
    if causal:
        i, j = torch.arange(Sq, device="cuda")[:, None], torch.arange(Sk, device="cuda")[None, :]
        s = s.masked_fill(j > i + (Sk - Sq), float("-inf"))
    o_ref = (s.softmax(-1) @ vh).transpose(1, 2).reshape(B * Sq, Hq * hd)
    o_ref.backward(do.float())
    o = L.attention(q, k, v, Hq, Hkv, hd, B, Sq, Sk, causal=causal)
    dq, dk, dv = K.attention_bwd(q, k, v, o, do, Hq, Hkv, hd, B, Sq, Sk, causal=causal)
    assert _rel(dq, qf.grad) < 1.5e-2 and _rel(dk, kf.grad) < 1.5e-2 and _rel(dv, vf.grad) < 1.5e-2
    if Sq == Sk and Hq == Hkv:   # column slices of one packed [rows, 3D] projection, as the training schedule passes them
        D = Hq * hd
        qkv = torch.cat((q, k, v), dim=1)
        dq2, dk2, dv2 = K.attention_bwd(qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:], o, do, Hq, Hkv, hd, B, Sq, Sk, causal=causal)
        assert torch.equal(dq2, dq) and torch.equal(dk2, dk) and torch.equal(dv2, dv)


@pytest.mark.parametrize("M,No,Ko", [(98304, 1536, 384), (6144, 384, 1152), (1000, 384, 200), (777, 392, 64), (64, 128, 128),
                                      (130, 8, 2048), (12288, 2048, 384)])
def test_wgrad_in_place_operands(M, No, Ko):
    """dW = dY^T X with both operands read in place as MN-major UMMA tiles and the rows split over CTAs (wgrad_tn.cu), vs fp32
    PyTorch on the same bf16 operands; strided operand views (column slices of a wider buffer) and accumulation."""
    from internnav_b200 import _bwd as K
    torch.manual_seed(M + No + Ko)
    dy = torch.randn(M, No, device="cuda").bfloat16()
    x = torch.randn(M, Ko, device="cuda").bfloat16()
    ref = dy.float().t() @ x.float()
    out = K.wgrad(dy, x)
    assert out.shape == (No, Ko) and _rel(out, ref) < 1e-3, _rel(out, ref)
    assert torch.equal(K.wgrad(dy, x), out)                      # fixed summation order: bit-reproducible
    wide_y = torch.randn(M, No + 16, device="cuda").bfloat16()
    wide_x = torch.randn(M, 2 * Ko + 8, device="cuda").bfloat16()
    o2 = K.wgrad(wide_y[:, 8:8 + No], wide_x[:, Ko:2 * Ko])
    assert _rel(o2, wide_y[:, 8:8 + No].float().t() @ wide_x[:, Ko:2 * Ko].float()) < 1e-3
    acc = torch.ones(No, Ko, device="cuda")
    K.wgrad(dy, x, out=acc, accumulate=True)
    assert _rel(acc, ref + 1.0) < 1e-3


def test_adamw_matches_torch():
    from internnav_b200 import _bwd as K
    torch.manual_seed(3)
    n = 100003
    p0 = torch.randn(n, device="cuda")
    ref = torch.nn.Parameter(p0.clone())
    opt = torch.optim.AdamW([ref], lr=1e-3, betas=(0.9, 0.95), eps=1e-8, weight_decay=0.1)
    master, m, v = p0.clone(), torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    work = torch.empty(n, device="cuda", dtype=torch.bfloat16)
    for step in range(1, 4):
        g = torch.randn(n, device="cuda")
        ref.grad = g.clone()
        opt.step()
        K.adamw(master, work, g, m, v, 1e-3, betas=(0.9, 0.95), eps=1e-8, weight_decay=0.1, step=step)
        assert _rel(master, ref.data) < 1e-6
        assert torch.equal(work, master.bfloat16())


def test_s2_training_forward_and_latent_query_gradient():
    """System-2 half of the training step on the GPU: TRAJ states and d loss / d latent_queries vs the oracle (padded-batch
    forward + autograd), tiny config, ragged prompts."""
    import numpy as np
    from internnav_b200.qwen import System2
    from oracle import qwen_oracle as Q
    cfg = Q.tiny_cfg()
    sd = Q.make_s2_state_dict(cfg, seed=10, vocab_rows=256)
    s2 = System2(cfg, device="cuda:0")
    s2.load_state_dict(sd)
    rng = np.random.Generator(np.random.PCG64(41))
    gpp = [[(1, 8, 12)], [(1, 4, 8), (1, 4, 4)], [(1, 4, 4)]]
    prompts = [Q.make_prompt(rng, 4 + 5 * i, gs, 13 - 4 * i) for i, gs in enumerate(gpp)]
    grids = [g for gs in gpp for g in gs]
    px = torch.randn(sum(t * h * w for t, h, w in grids), 1176, generator=torch.Generator().manual_seed(6)).bfloat16()
    G = torch.randn(len(prompts), cfg["n_query"], cfg["hidden"], generator=torch.Generator().manual_seed(7))
    states = s2.train_forward(prompts, px.cuda(), grids)
    grad = s2.train_backward(G.cuda())
    rows = [list(p) + [Q.TRAJ_TOKEN_INDEX] * 4 for p in prompts]
    S = max(len(r) for r in rows)
    ids = torch.tensor([r + [151643] * (S - len(r)) for r in rows])
    mask, t_s_pos = ids.ne(151643), [len(p) for p in prompts]
    with torch.no_grad():
        ref_states = Q.training_traj_states(sd, cfg, ids, mask, px.float(), grids, t_s_pos)
    ref_grad = Q.latent_query_grads(sd, cfg, ids, mask, px.float(), grids, t_s_pos, G.bfloat16().float())
    e_s, e_g = _rel(states.cpu(), ref_states), _rel(grad.cpu(), ref_grad)
    print("S2 train: states rel err", e_s, "latent_queries grad rel err", e_g)
    assert e_s < 2e-2 and e_g < 2e-2
    # and the states equal the inference latent plan of the same prompts (same kernels, different chunking)
    assert _rel(states, s2.generate_latents(prompts, px.cuda(), grids)) < 5e-3


def test_dual_system_training_step_vs_oracle():
    """End to end on the GPU: collated batch -> S2 TRAJ states -> S1 forward / backward -> latent_queries gradient, against
    the oracle chain (padded-batch decoder + autograd through the restated System 1); then one AdamW step moves the
    masters in the direction torch.optim.AdamW moves them."""
    import numpy as np
    from internnav_b200.internvla_n1 import InternVLAN1ForCausalLM
    from internnav_b200.manifest import random_navdp_state_dict
    from internnav_b200.train_step import DualSystemTrainer
    from internnav_b200.training import collate_traj_batch
    from oracle import navdp_oracle as O, qwen_oracle as Q
    cfg = Q.tiny_cfg()
    s2_sd = Q.make_s2_state_dict(cfg, seed=31, vocab_rows=512)
    s1_sd = {k: v.float() for k, v in random_navdp_state_dict(seed=32, vlm_token_dim=cfg["hidden"]).items()}
    model = InternVLAN1ForCausalLM(cfg, device="cuda:0")
    model.load_parts(s2_sd, s1_sd)
    rng = np.random.Generator(np.random.PCG64(33))
    g = torch.Generator().manual_seed(34)
    gpp, frames = [[(1, 8, 12)], [(1, 4, 8)]], [2, 1]
    inst = []
    for gs, f in zip(gpp, frames):
        ids = torch.tensor([Q.make_prompt(rng, 6, gs, 11)])
        n_p = sum(t * h * w for t, h, w in gs)
        inst.append(dict(input_ids=ids, labels=torch.full_like(ids, -100), pixel_values=torch.randn(n_p, 1176, generator=g).bfloat16(),
                         image_grid_thw=torch.tensor(gs), traj_images=torch.rand(f, 224, 224, 3, generator=g),
                         traj_depths=torch.rand(f, 224, 224, generator=g) * 5, traj_poses=torch.randn(f, 32, 3, generator=g) * 0.5))
    batch = collate_traj_batch(inst)
    B, fmax = len(inst), max(frames)
    noise = torch.randn(B * fmax, 32, 3, generator=g)
    ts = torch.randint(0, 20, (B * fmax,), generator=g)
    tr = DualSystemTrainer(model, s1_sd, s2_sd["model.latent_queries"], lr=1e-3)
    loss, grads, hs = tr.loss_and_grads(batch, noise, ts)
    # oracle chain on the CPU (fp32)
    with torch.no_grad():
        hs_ref = Q.training_traj_states(s2_sd, cfg, batch["input_ids"], batch["attention_mask"], batch["pixel_values"].float(),
                                        batch["image_grid_thw"], batch["t_s_pos"])
    loss_ref, grads_ref, dhs_ref = O.s1_training_grads(s1_sd, hs_ref, batch["traj_images"], batch["traj_depths"],
                                                       batch["traj_poses"], batch["video_frame_num"], noise, ts)
    glat_ref = Q.latent_query_grads(s2_sd, cfg, batch["input_ids"], batch["attention_mask"], batch["pixel_values"].float(),
                                    batch["image_grid_thw"], batch["t_s_pos"], dhs_ref)
    print("train step: loss", float(loss), "oracle", float(loss_ref), "TRAJ states rel", _rel(hs.cpu(), hs_ref))
    assert abs(float(loss) - float(loss_ref)) / float(loss_ref) < 1e-2
    bad = []
    for k, gr in grads_ref.items():
        rel = _rel(grads[k].cpu().reshape(gr.shape), gr)
        if rel > 0.08 and float(gr.norm()) > 1e-6:
            bad.append((k, rel))
    print("parameter gradients beyond 8 %:", bad[:10], "of", len(grads_ref))
    assert len(bad) <= len(grads_ref) // 50
    assert _rel(grads["model.latent_queries"].cpu(), glat_ref) < 0.1
    before = {k: v.clone() for k, v in list(tr.masters.items())[:5]}
    tr.step(batch, noise, ts)
    assert tr.steps == 1 and any(not torch.equal(before[k], tr.masters[k]) for k in before if k in tr.buckets.grads)
    # the CUDA-graph replay of the System-1 forward / backward computes the same step: two trainers from identical state,
    # one eager and one graphed, two steps each -> identical loss and masters (bit for bit: same kernels, same order)
    ta = DualSystemTrainer(model, s1_sd, s2_sd["model.latent_queries"], lr=1e-3, max_grad_norm=1.0)
    tb = DualSystemTrainer(model, s1_sd, s2_sd["model.latent_queries"], lr=1e-3, max_grad_norm=1.0, graph_s1=True)
    dev_batch = {k: (v.cuda() if torch.is_tensor(v) and k in ("traj_images", "traj_depths", "traj_poses", "video_frame_num")
                     else v) for k, v in batch.items()}
    model._s2.set_latent_queries(ta.latent)          # `tr.step` above left ITS updated queries in the shared handle
    for _ in range(2):
        la = float(ta.step(dev_batch, noise.cuda(), ts.cuda()))
        model._s2.set_latent_queries(tb.latent)      # both trainers drive the same System-2 handle
        lb = float(tb.step(dev_batch, noise.cuda(), ts.cuda()))
        model._s2.set_latent_queries(ta.latent)
        assert abs(la - lb) <= 1e-6 * max(1.0, abs(la)), (la, lb)
    worst = max(float((ta.masters[k] - tb.masters[k]).abs().max()) for k in ta.masters)
    assert worst < 1e-6, worst
