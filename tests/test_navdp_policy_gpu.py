"""Stand-alone NavDP policy (SURVEY.md §8f-3) on the GPU: `internnav_b200.navdp_policy.NavDPNet` (libn1b200.so) against the
fp32 oracle (oracle/navdp_policy_oracle.py, pinned to the reference's own NavDPNet), with the bf16-eager run of the same
oracle as the reference-equivalent bound.  Tolerance: rel-L2 <= 2e-2 and <= 2 x bf16 eager (+ 2e-3)."""
import pytest
import torch

pytestmark = pytest.mark.gpu
TOL = 2e-2


def _rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-12)).item()


@pytest.fixture(scope="module")
def env():
    from internnav_b200.manifest import random_navdp_policy_state_dict
    from internnav_b200.navdp_policy import NavDPNet
    torch.backends.cuda.matmul.allow_tf32 = False
    sd = random_navdp_policy_state_dict(seed=7)
    m = NavDPNet(device="cuda:0")
    m.load_state_dict(sd)
    sd_gpu = {k: v.cuda() for k, v in sd.items()}
    return m, sd_gpu, {k: v.bfloat16() for k, v in sd_gpu.items()}


def _inputs(B, Ns, seed):
    g = torch.Generator().manual_seed(seed)
    return dict(images=torch.rand(B, 8, 224, 224, 3, generator=g).cuda(), depths=(torch.rand(B, 1, 224, 224, 1, generator=g) * 5).cuda(),
                goal=torch.randn(B, 3, generator=g).cuda(), x_init=torch.randn(B * Ns, 24, 3, generator=g).cuda(),
                step_noise=torch.randn(9, B * Ns, 24, 3, generator=g).cuda())


def test_stages_vs_oracle(env):
    from oracle import navdp_oracle as O, navdp_policy_oracle as P
    m, sd, sdb = env
    inp = _inputs(2, 32, 3)
    rgbd = m.rgbd_encoder(inp["images"], inp["depths"])
    with torch.no_grad():
        ref = P.rgbd_backbone(sd, inp["images"], inp["depths"])
        eag = P.rgbd_backbone(sdb, inp["images"].bfloat16(), inp["depths"].bfloat16())
    e, ee = _rel(rgbd, ref), _rel(eag, ref)
    print("memory tokens rel err", e, "bf16 eager", ee)
    assert e < TOL and e < 2 * ee + 2e-3, (e, ee)
    goal = m.point_encoder(inp["goal"]).unsqueeze(1)
    with torch.no_grad():
        goal_ref = O._lin(sd, "point_encoder", inp["goal"]).unsqueeze(1)
        assert _rel(goal, goal_ref) < 1e-5
        k = torch.tensor([6])
        eps_ref = P.predict_noise(sd, inp["x_init"], k.cuda(), goal_ref, ref)
        eps_eag = P.predict_noise(sdb, inp["x_init"].bfloat16(), k.cuda(), goal_ref.bfloat16(), ref.bfloat16())
        cr_ref = P.predict_critic(sd, inp["x_init"], ref)
        cr_eag = P.predict_critic(sdb, inp["x_init"].bfloat16(), ref.bfloat16())
    eps = m.predict_noise(inp["x_init"], k, goal_ref.bfloat16(), ref.bfloat16())
    e, ee = _rel(eps, eps_ref), _rel(eps_eag, eps_ref)
    print("eps rel err", e, "bf16 eager", ee)
    assert e < TOL and e < 2 * ee + 2e-3, (e, ee)
    cr = m.predict_critic(inp["x_init"], ref.bfloat16())
    # the critic is a scalar per sample (a mean over T of a 384-wide projection): judge it on the centred values
    e = _rel(cr - cr.mean(), cr_ref - cr_ref.mean())
    ee = _rel(cr_eag.float() - cr_eag.float().mean(), cr_ref - cr_ref.mean())
    print("critic rel err (centred)", e, "bf16 eager", ee)
    assert e < 5e-2 and e < 2 * ee + 5e-3, (e, ee)


def test_entry_points_vs_oracle(env):
    from oracle import navdp_policy_oracle as P
    m, sd, sdb = env
    inp = _inputs(1, 32, 4)
    neg, pos = m.predict_pointgoal_batch_action_vel(inp["goal"], inp["images"], inp["depths"], sample_num=32,
                                                    x_init=inp["x_init"], step_noise=inp["step_noise"])
    assert neg.shape == (8, 24, 3) and pos.shape == (8, 24, 3)
    with torch.no_grad():
        r_neg, r_pos, x_ref, cr_ref = P.predict_pointgoal_batch_action_vel(sd, inp["goal"], inp["images"], inp["depths"],
                                                                           inp["x_init"], inp["step_noise"])
        _, _, x_eag, _ = P.predict_pointgoal_batch_action_vel(sdb, inp["goal"].bfloat16(), inp["images"].bfloat16(),
                                                              inp["depths"].bfloat16(), inp["x_init"].bfloat16(),
                                                              inp["step_noise"].bfloat16())
    # the sampled trajectories before ranking
    goal = m.point_encoder(inp["goal"]).unsqueeze(1).bfloat16()
    x = m.sample(goal, m.rgbd_encoder(inp["images"], inp["depths"]), inp["x_init"], inp["step_noise"], num_steps=10)
    e, ee = _rel(x, x_ref), _rel(x_eag, x_ref)
    print("10-step trajectories rel err", e, "bf16 eager", ee)
    # 10 chained denoising steps x 16 layers: the reference-equivalent bf16-eager run itself can sit above the 2e-2
    # single-pass bar; as in test_full_config_gpu.py the bar is 3e-2 AND no worse than bf16 eager
    assert e < 3e-2 and e < ee + 2e-3, (e, ee)
    # ranking: the 8 best / worst of ours are a selection of our own critic values (consistency) and largely the oracle's
    traj_ref = torch.cumsum(x_ref / 4.0, dim=1)

    def members(sel, pool):
        return {int(((pool - t).flatten(1).norm(dim=1)).argmin()) for t in sel}
    ours_pos, ref_pos = members(pos.float(), torch.cumsum(x.float() / 4.0, dim=1)), members(r_pos, traj_ref)
    print("top-8 overlap with the fp32 oracle:", len(ours_pos & ref_pos), "of 8")
    assert len(ours_pos) == 8 and len(ours_pos & ref_pos) >= 5
    neg2, pos2 = m.predict_nogoal_batch_action_vel(inp["images"], inp["depths"], sample_num=32, x_init=inp["x_init"],
                                                   step_noise=inp["step_noise"])
    assert neg2.shape == (8, 24, 3) and torch.isfinite(pos2).all() and not torch.equal(pos2, pos)
