"""Parity AT THE BENCHMARKED CONFIGURATION (BASELINE.json configs[2] / configs[3]) -- VERDICT r1 "what's weak" #1.

  (i)   one environment through the full-depth Qwen2.5-VL-7B shapes (32 vision blocks, 28 decoder layers, S = 304) against
        the fp32 oracle run on the same GPU, with the bf16-eager run of the same oracle as the reference-equivalent bound;
  (ii)  the B = 64 batched calls equal 64 single-environment calls bit for bit (environment independence), for System 2
        (latents) and for System 1 (trajectories) -- (i) + (ii) together are parity of the batched benchmark step;
  (iii) two host threads drive the same handles concurrently (S2 on one stream / workspace, S1 on another), as the
        reference agent does (internvla_n1_agent.py L133-208), and reproduce the single-threaded results bit for bit.

Tolerance (SURVEY.md §8d): rel-L2 vs the fp32 oracle <= 2x the bf16-eager error (+ 2e-3 slack) and <= 2e-2 -- except
that at FULL DEPTH with random weights the reference-equivalent bf16-eager run itself can sit above the
absolute bar, so there the absolute bar is 3e-2 and the binding requirement is that the
CUDA path is at least as accurate as bf16 eager."""
import threading

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
TOL = 2e-2
GRID = (1, 28, 28)          # one 392 x 392 frame: 784 patches -> 196 image tokens
N_PRE, N_POST = 12, 90      # 12 + (1 + 196 + 1) + 90 = 300 prompt tokens, + 4 latent queries = S 304 (bench.py)


def _rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-12)).item()


@pytest.fixture(scope="module")
def full():
    """Random-init weights of the full 7B shapes, generated on the device in fp32 (the oracle's copy, 33 GB) and packed
    into the library from the same tensors (bf16, 15.4 GB)."""
    from internnav_b200.manifest import random_s2_state_dict
    from internnav_b200.qwen import System2
    from oracle import qwen_oracle as Q
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    cfg = dict(Q.QWEN25VL_7B)
    sd = random_s2_state_dict(cfg, seed=11, device="cuda", dtype=torch.float32)
    s2 = System2(cfg, device="cuda:0")
    s2.load_state_dict(sd)
    return cfg, sd, s2


def _prompts(B, seed):
    from oracle import qwen_oracle as Q
    rng = np.random.Generator(np.random.PCG64(seed))
    return [Q.make_prompt(rng, N_PRE, [GRID], N_POST) for _ in range(B)]


def test_full_depth_one_env_vs_fp32_oracle(full):
    from oracle import qwen_oracle as Q
    cfg, sd, s2 = full
    prompts = _prompts(1, 3)
    assert len(prompts[0]) + cfg["n_query"] == 304
    px = torch.randn(784, 1176, generator=torch.Generator().manual_seed(5)).bfloat16().cuda()
    feats = s2.visual(px, [GRID])
    lat = s2.generate_latents(prompts, px, [GRID])
    sdb = {k: v.bfloat16() for k, v in sd.items()}
    with torch.no_grad():
        ref_v = Q.vit_forward(sd, cfg, px.float(), [GRID])
        eag_v = Q.vit_forward(sdb, cfg, px, [GRID])
        ids = torch.tensor([prompts[0]])
        ref_l = Q.generate_latents(sd, cfg, ids, px.float(), [GRID])
        eag_l = Q.generate_latents(sdb, cfg, ids, px, [GRID])
    e_v, ee_v = _rel(feats, ref_v), _rel(eag_v, ref_v)
    e_l, ee_l = _rel(lat[0], ref_l[0]), _rel(eag_l[0], ref_l[0])
    print("full depth (32 + 28 layers, S = 304): ViT rel err %.4f (bf16 eager %.4f); latents rel err %.4f (bf16 eager %.4f)"
          % (e_v, ee_v, e_l, ee_l))
    # 60 bf16 layers deep: the absolute bar is 3e-2 (see the module docstring); the binding bar is "no worse than the
    # reference-equivalent bf16-eager run"
    assert e_v < 3e-2 and e_v < ee_v + 2e-3, (e_v, ee_v)
    assert e_l < 3e-2 and e_l < ee_l + 2e-3, (e_l, ee_l)


def test_batch64_equals_64_single_env_calls_system2(full):
    cfg, sd, s2 = full
    B = 64
    prompts = _prompts(B, 17)
    px = torch.randn(B * 784, 1176, generator=torch.Generator().manual_seed(6)).bfloat16().cuda()
    batched = s2.generate_latents(prompts, px, [GRID] * B)
    assert batched.shape == (B, 4, 3584) and torch.isfinite(batched.float()).all()
    worst = 0.0
    for b in range(B):
        one = s2.generate_latents([prompts[b]], px[b * 784:(b + 1) * 784], [GRID])
        if not torch.equal(one[0], batched[b]):
            worst = max(worst, _rel(one[0], batched[b]))
    print("S2 batched vs single-env: worst rel difference", worst)
    assert worst == 0.0, "batched latents differ from the single-environment calls (rel %.3e)" % worst


def test_batch64_equals_64_single_env_calls_system1():
    from internnav_b200.manifest import random_navdp_state_dict
    from internnav_b200.navdp import NavDP_Policy_DPT_CriticSum_DAT
    m = NavDP_Policy_DPT_CriticSum_DAT(memory_size=2, predict_size=32, navdp_version=0.1, device="cuda:0")
    m.load_state_dict(random_navdp_state_dict(seed=3))
    B, Ns, T, K = 64, 32, 32, 20
    g = torch.Generator().manual_seed(8)
    lat = torch.randn(B, 4, 3584, generator=g).bfloat16().cuda()
    rgb = torch.rand(B, 2, 224, 224, 3, generator=g).cuda()
    dep = (torch.rand(B, 2, 224, 224, 1, generator=g) * 5).cuda()
    x0 = torch.randn(B * Ns, T, 3, generator=g).cuda()
    nz = torch.randn(K - 1, B * Ns, T, 3, generator=g).cuda()
    batched = m.predict_pointgoal_action_async(lat, rgb, dep, x_init=x0, step_noise=nz)
    worst = 0.0
    for b in range(B):
        sl = slice(b * Ns, (b + 1) * Ns)
        one = m.predict_pointgoal_action_async(lat[b:b + 1], rgb[b:b + 1], dep[b:b + 1], x_init=x0[sl].contiguous(),
                                               step_noise=nz[:, sl].contiguous())
        if not torch.equal(one, batched[sl]):
            worst = max(worst, _rel(one, batched[sl]))
    print("S1 batched vs single-env: worst rel difference", worst)
    assert worst == 0.0, "batched trajectories differ from the single-environment calls (rel %.3e)" % worst


def test_two_host_threads_share_the_handles(full):
    """S2 on thread A (its own stream and workspace), S1 on thread B, 6 rounds each, concurrently -- every result equals
    the single-threaded one (the C ABI promises this: include/n1b200.h, 'concurrent calls with separate workspaces')."""
    from internnav_b200.manifest import random_navdp_state_dict
    from internnav_b200.navdp import NavDP_Policy_DPT_CriticSum_DAT
    cfg, sd, s2 = full
    m = NavDP_Policy_DPT_CriticSum_DAT(memory_size=2, predict_size=32, navdp_version=0.1, device="cuda:0")
    m.load_state_dict(random_navdp_state_dict(seed=4))
    B = 4
    g = torch.Generator().manual_seed(9)
    prompt_sets = [_prompts(B, 100 + r) for r in range(6)]
    px = torch.randn(B * 784, 1176, generator=g).bfloat16().cuda()
    lat = torch.randn(B, 4, 3584, generator=g).bfloat16().cuda()
    rgb = torch.rand(B, 2, 224, 224, 3, generator=g).cuda()
    dep = (torch.rand(B, 2, 224, 224, 1, generator=g) * 5).cuda()
    x0 = torch.randn(B * 32, 32, 3, generator=g).cuda()
    nz = torch.randn(19, B * 32, 32, 3, generator=g).cuda()
    ref_s2 = [s2.generate_latents(p, px, [GRID] * B).clone() for p in prompt_sets]
    ref_s1 = m.predict_pointgoal_action_async(lat, rgb, dep, x_init=x0, step_noise=nz).clone()
    torch.cuda.synchronize()
    out, err = {"s2": [], "s1": []}, []

    def run_s2():
        try:
            st = torch.cuda.Stream()
            with torch.cuda.stream(st):
                for p in prompt_sets:
                    out["s2"].append(s2.generate_latents(p, px, [GRID] * B).clone())
                st.synchronize()
        except Exception as e:  # noqa: BLE001
            err.append(e)

    def run_s1():
        try:
            st = torch.cuda.Stream()
            with torch.cuda.stream(st):
                for _ in range(6):
                    out["s1"].append(m.predict_pointgoal_action_async(lat, rgb, dep, x_init=x0, step_noise=nz).clone())
                st.synchronize()
        except Exception as e:  # noqa: BLE001
            err.append(e)

    ta, tb = threading.Thread(target=run_s2), threading.Thread(target=run_s1)
    ta.start(), tb.start()
    ta.join(120), tb.join(120)
    assert not ta.is_alive() and not tb.is_alive(), "a worker thread did not finish"
    assert not err, err
    torch.cuda.synchronize()
    assert len(out["s2"]) == 6 and len(out["s1"]) == 6
    for r in range(6):
        assert torch.equal(out["s2"][r], ref_s2[r]), "S2 result of round %d changed under concurrency" % r
        assert torch.equal(out["s1"][r], ref_s1), "S1 result of round %d changed under concurrency" % r
