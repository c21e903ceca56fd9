"""NextDiT System 1 (internnav_b200/nextdit.py, f1) on the GPU against (a) the committed output of the REFERENCE's own
generate_traj (tests/golden/nextdit_reference.npz, see tests/test_oracle_nextdit.py for what that pins) and (b) the fp32
oracle run on the same device, with the bf16-eager run of the same oracle as the reference-equivalent bound.

Tolerance (SURVEY.md §8d): rel-L2 <= 2e-2 and <= 2x bf16 eager (+2e-3) for single passes; the 10 chained Euler steps
x 12 blocks meet the same bar against the oracle; against the reference-run fixture (fp32) the bar is 3e-2."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "nextdit_reference.npz")


def _rel(a, b):
    a, b = a.float().cpu(), torch.as_tensor(b).float().cpu()
    return float((a - b).norm() / (b.norm() + 1e-12))


@pytest.fixture(scope="module")
def env():
    from internnav_b200.manifest import random_nextdit_state_dict
    from internnav_b200.nextdit import NextDiTSystem1
    g = np.load(GOLD)
    sd = random_nextdit_state_dict(int(g["seed"]))
    m = NextDiTSystem1(device="cuda:0").load_state_dict(sd)
    sdc = {k: v.cuda() for k, v in sd.items()}
    sdb = {k: v.bfloat16() for k, v in sdc.items()}
    return m, sdc, sdb, g


def test_against_the_reference_run(env):
    from oracle.gen_golden_nextdit import make_inputs
    m, sdc, sdb, g = env
    inp = make_inputs(int(g["seed"]), int(g["batch"]), int(g["ns"]))
    cond = m.condition_tokens(inp["traj_latents"].cuda(), inp["images_dp"].cuda())
    e = _rel(cond, g["condition_tokens"])
    print("condition tokens vs the reference run:", e)
    assert e < 2e-2
    for scale, key, exact in ((1.0, "traj_scale_1", False), (1.0, "traj_scale_1", True), (2.5, "traj_scale_2p5", False)):
        out = m.generate_traj(inp["traj_latents"].cuda(), inp["images_dp"].cuda(), guidance_scale=scale,
                              num_sample_trajs=int(g["ns"]), x_init=inp["x_init"].cuda(), exact_cfg=exact)
        assert out.shape == (3, 32, 3) and torch.isfinite(out).all()
        e = _rel(out, g[key])
        print("trajectories vs the reference run, guidance %.1f exact_cfg=%s:" % (scale, exact), e)
        assert e < 3e-2, (scale, exact, e)


def test_batched_vs_oracle_and_eager(env):
    from oracle import nextdit_oracle as O
    m, sdc, sdb, _ = env
    B, Ns = 3, 4
    gen = torch.Generator().manual_seed(21)
    lat = torch.randn(B, 4, 3584, generator=gen).cuda()
    img = torch.rand(B, 2, 224, 224, 3, generator=gen).cuda()
    x0 = torch.randn(B * Ns, 32, 3, generator=gen).bfloat16().float().cuda()
    with torch.no_grad():
        c_ref = O.condition_tokens(sdc, lat, img)
        c_eag = O.condition_tokens(sdb, lat.bfloat16(), img)
    cond = m.condition_tokens(lat.bfloat16(), img)
    e, ee = _rel(cond, c_ref), _rel(c_eag, c_ref)
    print("condition tokens rel err", e, "bf16 eager", ee)
    assert e < 2e-2 and e < 2 * ee + 2e-3, (e, ee)
    # one evaluation of the DiT + decoder from the same condition tokens (first Euler step, guidance batch)
    ts, sig = O.flow_match_schedule(10)
    with torch.no_grad():
        hid = torch.cat((torch.zeros_like(c_ref), c_ref), 0).repeat_interleave(Ns, dim=0)
        feats = O.action_features(sdc, x0).repeat(2, 1, 1)
        tt = ts[0].expand(feats.shape[0]).to(torch.long).cuda()
        p_ref = O._lin(sdc, "action_decoder", O.traj_dit(sdc, feats, tt, hid))
        p_eag = O._lin(sdb, "action_decoder", O.traj_dit(sdb, O.action_features(sdb, x0.bfloat16()).repeat(2, 1, 1), tt, hid.bfloat16()))
    from internnav_b200 import _lib
    z = torch.cat((torch.zeros_like(c_ref), c_ref), 0).bfloat16()
    mods, so, kn, kv = m._conditioning(z, m.schedule(10)[0])
    x = torch.empty(2 * B * Ns * 32, 384, device="cuda", dtype=torch.bfloat16)
    for h in range(2):
        _lib.action_embed(x0.contiguous(), m.w["enc.w"], m.w["enc.b"], m._pos(32), out=x[h * B * Ns * 32:(h + 1) * B * Ns * 32])
    pred = m._dit_step(x, mods[0], so[0], kn, kv, Ns * 32, 2 * B * Ns, 32, 36, Ns)[:, :3].reshape(p_ref.shape)
    e, ee = _rel(pred, p_ref), _rel(p_eag, p_ref)
    print("one DiT evaluation rel err", e, "bf16 eager", ee)
    assert e < 2e-2 and e < 2 * ee + 2e-3, (e, ee)
    # the whole sampler, both guidance modes
    for scale in (1.0, 3.0):
        with torch.no_grad():
            t_ref = O.generate_traj(sdc, lat, img, x0, guidance_scale=scale, num_sample_trajs=Ns)
            t_eag = O.generate_traj(sdb, lat.bfloat16(), img, x0.bfloat16(), guidance_scale=scale, num_sample_trajs=Ns)
        out = m.generate_traj(lat.bfloat16(), img, guidance_scale=scale, num_sample_trajs=Ns, x_init=x0)
        e, ee = _rel(out, t_ref), _rel(t_eag, t_ref)
        print("10-step trajectories, guidance %.1f: rel err" % scale, e, "bf16 eager", ee)
        assert e < 2e-2 and e < 2 * ee + 2e-3, (scale, e, ee)


def test_environments_are_independent(env):
    """A batch of environments equals the single-environment calls bit for bit (the reference handles one per call)."""
    m = env[0]
    B, Ns = 4, 8
    gen = torch.Generator().manual_seed(4)
    lat = torch.randn(B, 4, 3584, generator=gen).bfloat16().cuda()
    img = torch.rand(B, 2, 224, 224, 3, generator=gen).cuda()
    x0 = torch.randn(B * Ns, 32, 3, generator=gen).bfloat16().cuda()
    full = m.generate_traj(lat, img, num_sample_trajs=Ns, x_init=x0, guidance_scale=2.0)
    eager = m.generate_traj(lat, img, num_sample_trajs=Ns, x_init=x0, guidance_scale=2.0, graph=False)
    assert torch.equal(full, eager), "the CUDA-graph replay of the sampler differs from the eager launch sequence"
    again = m.generate_traj(lat, img, num_sample_trajs=Ns, x_init=x0, guidance_scale=2.0)
    assert torch.equal(full, again)
    for b in range(B):
        one = m.generate_traj(lat[b:b + 1], img[b:b + 1], num_sample_trajs=Ns, x_init=x0[b * Ns:(b + 1) * Ns], guidance_scale=2.0)
        assert torch.equal(one, full[b * Ns:(b + 1) * Ns]), "environment %d differs in the batch" % b


def test_row_kernels():
    from internnav_b200 import _lib
    torch.manual_seed(0)
    rows, D, G = 96, 384, 3
    x = torch.randn(rows, D, device="cuda").bfloat16()
    res = torch.randn(rows, D, device="cuda").bfloat16()
    w = (1 + 0.1 * torch.randn(D, device="cuda")).float()
    mod = torch.randn(G, 4 * D, device="cuda").bfloat16()
    mg = mod[:, D:2 * D].float().repeat_interleave(rows // G, dim=0)
    xf = x.float()
    rms = xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-5) * w
    assert _rel(_lib.mod_norm(x, w, mod[:, D:2 * D], rows // G, 1e-5, _lib.MOD_RMS_SCALE), rms * (1 + mg)) < 4e-3
    ln = torch.nn.functional.layer_norm(xf, (D,), None, None, 1e-6)
    assert _rel(_lib.mod_norm(x, None, mod[:, D:2 * D], rows // G, 1e-6, _lib.MOD_LN_SCALE), ln * (1 + mg)) < 4e-3
    assert _rel(_lib.mod_norm(x, w, mod[:, D:2 * D], rows // G, 1e-5, _lib.MOD_GATED_RESIDUAL, residual=res),
                res.float() + torch.tanh(mg) * rms) < 4e-3
    assert torch.equal(_lib.add(x, res), (x.float() + res.float()).bfloat16())
    a = torch.randn(64, 384, device="cuda").bfloat16()
    wt = torch.randn(256, 384, device="cuda").bfloat16()
    ref = a.float() @ wt.float().t()
    assert _rel(_lib.gemm(a, wt, act=_lib.ACT_SILU), torch.nn.functional.silu(ref)) < 5e-3
    assert _rel(_lib.gemm(a, wt, act=_lib.ACT_GELU_TANH), torch.nn.functional.gelu(ref, approximate="tanh")) < 5e-3
