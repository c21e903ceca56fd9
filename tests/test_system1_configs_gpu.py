"""The System-2-only model and the synchronous NextDiT head on the GPU.

System 2 only: a checkpoint directory without `system1` and without latent_queries loads through from_pretrained; its
greedy tokens pass the teacher-forced check against the fp32 oracle (as tests/test_s2_gpu.py) and equal those of a dual
model with the same System-2 weights; every call that needs latent_queries returns the library's error; the policy runs
the same episode as with the dual model.  Synchronous head (`system1 = "nextdit"`): the reference's own run
(tests/golden/nextdit_sync_reference.npz), the fp32 oracle at the SURVEY.md §8d bar, batch independence, graph replay."""
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "nextdit_sync_reference.npz")
MARGIN = 0.15  # logit units, as tests/test_s2_gpu.py


def _rel(a, b):
    a, b = torch.as_tensor(a).float().cpu(), torch.as_tensor(b).float().cpu()
    return float((a - b).norm() / (b.norm() + 1e-12))


def _hf_config(cfg):
    return dict(architectures=["Qwen2_5_VLForConditionalGeneration"], model_type="qwen2_5_vl", hidden_size=cfg["hidden"],
                num_hidden_layers=cfg["layers"], num_attention_heads=cfg["heads"], num_key_value_heads=cfg["kv_heads"],
                intermediate_size=cfg["inter"], vocab_size=cfg["vocab"], rms_norm_eps=cfg["rms_eps"],
                rope_theta=cfg["rope_theta"], rope_scaling={"type": "mrope", "mrope_section": cfg["mrope"]},
                vision_config=dict(depth=cfg["v_depth"], hidden_size=cfg["v_hidden"], num_heads=cfg["v_heads"],
                                   intermediate_size=cfg["v_inter"], out_hidden_size=cfg["v_out"], patch_size=cfg["v_patch"],
                                   temporal_patch_size=cfg["v_tpatch"], spatial_merge_size=cfg["v_merge"],
                                   window_size=cfg["v_window"], fullatt_block_indexes=cfg["fullatt"]))


@pytest.fixture(scope="module")
def models(tmp_path_factory):
    """(System-2-only model from a checkpoint directory, dual model with the same System-2 weights, cfg, fp32 sd)."""
    from safetensors.torch import save_file
    from internnav_b200.internvla_n1 import InternVLAN1ForCausalLM
    from oracle import qwen_oracle as Q
    torch.backends.cuda.matmul.allow_tf32 = False
    cfg = Q.tiny_cfg()
    sd = Q.make_s2_state_dict(cfg, seed=5, lm_head=True)
    path = tmp_path_factory.mktemp("system2_ckpt")
    save_file({k: v.contiguous() for k, v in sd.items() if k != "model.latent_queries"}, str(path / "model.safetensors"))
    (path / "config.json").write_text(json.dumps(_hf_config(cfg)))
    s2only = InternVLAN1ForCausalLM.from_pretrained(str(path), torch_dtype=torch.bfloat16, device_map={"": "cuda:0"})
    dual = InternVLAN1ForCausalLM(cfg, device="cuda:0", system1="navdp_async")
    dual._s2.load_state_dict(sd)   # System 2 of the dual model; no System-1 call is made here
    return s2only, dual, cfg, {k: v.cuda() for k, v in sd.items()}


def _inputs(cfg, seed=3):
    from oracle import qwen_oracle as Q
    rng = np.random.Generator(np.random.PCG64(seed))
    gpp = [[(1, 8, 12)], [(1, 16, 16), (1, 4, 4)], [(1, 4, 8)]]
    prompts = [Q.make_prompt(rng, 6 + 2 * i, gs, 10 + 3 * i) for i, gs in enumerate(gpp)]
    grids = [g for gs in gpp for g in gs]
    px = torch.randn(sum(t * h * w for t, h, w in grids), 1176, generator=torch.Generator().manual_seed(seed)).bfloat16().cuda()
    return prompts, gpp, grids, px


def test_system2_only_generate_matches_the_oracle_and_the_dual_model(models):
    from oracle import qwen_oracle as Q
    s2only, dual, cfg, sd = models
    assert s2only.get_system1_type() is None and not s2only._s2.has_latent_queries and dual._s2.has_latent_queries
    prompts, gpp, grids, px = _inputs(cfg)
    out = s2only.generate(prompts, px, grids, max_new_tokens=8, return_dict_in_generate=True)
    ref = dual.generate(prompts, px, grids, max_new_tokens=8, return_dict_in_generate=True)
    both = dual.generate_with_latents(prompts, px, grids, max_new_tokens=8)
    assert out.generated == ref.generated == both.generated and torch.equal(out.sequences, ref.sequences)
    exact = total = off = 0
    for b, (ids, gs) in enumerate(zip(prompts, gpp)):
        n = sum(t * h * w for t, h, w in gs)
        cur = torch.tensor([ids])
        with torch.no_grad():
            feats = Q.vit_forward(sd, cfg, px[off:off + n].float(), gs)
            for tok in out.generated[b]:
                lg = Q.next_token_logits(sd, cfg, cur, feats, gs)
                assert float(lg.max() - lg[tok]) <= MARGIN, (b, tok, int(lg.argmax()))
                exact += int(int(lg.argmax()) == tok)
                total += 1
                cur = torch.cat([cur, torch.tensor([[tok]])], dim=1)
        off += n
    assert exact >= 0.6 * total, (exact, total)
    # the greedy tokens of the first prompt against the oracle's own greedy_generate
    with torch.no_grad():
        g0 = Q.greedy_generate(sd, cfg, torch.tensor([prompts[0]]), px[:96].float(), gpp[0], max_new_tokens=8)
    print("system-2-only greedy", out.generated[0], "oracle", g0, "exact", exact, "/", total)
    assert out.generated[0] == g0


def test_calls_that_need_latent_queries_return_errors(models):
    from internnav_b200._lib import N1Error
    s2only, _, cfg, _ = models
    prompts, _, grids, px = _inputs(cfg, 4)
    before = s2only.generate(prompts, px, grids, max_new_tokens=4, return_dict_in_generate=True).generated
    s2 = s2only._s2
    for call in (lambda: s2.generate_latents(prompts, px, grids),                          # TRAJ-token (latent) plan
                 lambda: s2.generate(prompts, px, grids, max_new_tokens=4, with_latents=True),
                 lambda: s2.set_latent_queries(torch.zeros(4, cfg["hidden"], device="cuda")),
                 lambda: s2.train_forward(prompts, px, grids)):
        with pytest.raises(N1Error, match="latent_queries"):
            call()
    for call in (lambda: s2only.generate_latents(prompts, px, grids), lambda: s2only.generate_with_latents(prompts, px, grids)):
        with pytest.raises(RuntimeError, match="System 1"):
            call()
    assert s2only.generate(prompts, px, grids, max_new_tokens=4, return_dict_in_generate=True).generated == before


class _Forward:
    """The model behind the policy, recording (prompts, generated) of every call; make_kv_pool only with `pool`."""

    def __init__(self, model, pool):
        self.m, self.config, self.device, self.has_system1, self.calls = model, model.config, model.device, model.has_system1, []
        self.make_feature_pool = model.make_feature_pool
        if pool:
            self.make_kv_pool = model.make_kv_pool

    def _rec(self, out, prompts):
        self.calls.append((prompts, out.generated))
        return out

    def generate(self, prompts, *a, **kw):
        return self._rec(self.m.generate(prompts, *a, **kw), prompts)

    def generate_with_latents(self, prompts, *a, **kw):
        return self._rec(self.m.generate_with_latents(prompts, *a, **kw), prompts)


@pytest.mark.parametrize("pool,vision_cache", [(False, 0), (True, 0), (True, 2), (False, 2)])
def test_policy_episode_matches_the_dual_model(models, pool, vision_cache):
    from internnav_b200.policy import InternVLAN1Policy
    from test_policy_kv_gpu import LookDownProcessor, _frame

    class Proc(LookDownProcessor):   # answers alternate between look-down actions and pixel goals
        class _Tok(LookDownProcessor._Tok):
            n = 0

            def decode(self, ids, skip_special_tokens=True):
                s = LookDownProcessor._Tok.decode(self, ids)
                self.n += 1
                return s if self.n % 2 else s[:-1] + " 12 34"

        def __init__(self):
            self.tokenizer = self._Tok()

    s2only, dual, _, _ = models
    fw = [_Forward(m, pool) for m in (s2only, dual)]
    pols = [InternVLAN1Policy(f, Proc(), num_envs=2, num_history=4, resize_w=112, resize_h=112, max_new_tokens=6,
                              vision_cache_frames=vision_cache) for f in fw]
    results = [[], []]
    for i, pol in enumerate(pols):
        for k in range(3):
            pol.step_no_infer([0, 1], [_frame(k, e) for e in (0, 1)])
        for envs, k, ld in (([0, 1], 3, [False, False]), ([0], 4, [True]), ([0, 1], 5, [False, False]), ([1], 6, [True])):
            res = pol.s2_step(envs, [_frame(k, e) for e in envs], None, None, ["go to door %d" % e for e in envs], None, ld)
            assert all(not isinstance(r, Exception) for r in res), res
            results[i] += res
    assert fw[0].calls == fw[1].calls and len(fw[0].calls) == 4
    pixel = 0
    for r0, r1 in zip(*results):
        assert r0.output_action == r1.output_action and r0.output_latent is None
        if r1.output_pixel is not None:
            pixel += 1
            assert np.array_equal(r0.output_pixel, r1.output_pixel) and r1.output_latent is not None
    assert pixel == 3
    with pytest.raises(RuntimeError, match="System 1"):
        pols[0].s1_step_latent([0], [torch.zeros(1, 2, 224, 224, 3)], [torch.zeros(1, 2, 224, 224, 1)],
                               [torch.zeros(1, 4, 256)])


# ------------------------------------------------------------------------------------------------ synchronous NextDiT
@pytest.fixture(scope="module")
def head():
    from internnav_b200.manifest import random_nextdit_state_dict
    from internnav_b200.nextdit import NextDiTSystem1
    g = np.load(GOLD)
    sd = random_nextdit_state_dict(int(g["seed"]), asynchronous=False)
    m = NextDiTSystem1(device="cuda:0", asynchronous=False).load_state_dict(sd)
    return m, {k: v.cuda() for k, v in sd.items()}, g


def test_sync_head_against_the_reference_run(head):
    from oracle.gen_golden_nextdit import make_inputs
    m, _, g = head
    inp = make_inputs(int(g["seed"]), int(g["batch"]), int(g["ns"]))
    cond = m.condition_tokens(inp["traj_latents"].cuda(), None)
    assert cond.shape == (1, 4, 768) and _rel(cond, g["condition_tokens"]) < 2e-2
    for scale, key, exact in ((1.0, "traj_scale_1", False), (1.0, "traj_scale_1", True), (2.5, "traj_scale_2p5", False)):
        out = m.generate_traj(inp["traj_latents"].cuda(), inp["images_dp"].cuda(), guidance_scale=scale,
                              num_sample_trajs=int(g["ns"]), x_init=inp["x_init"].cuda(), exact_cfg=exact)
        e = _rel(out, g[key])
        print("sync head vs the reference run, guidance %.1f exact_cfg=%s:" % (scale, exact), e)
        assert out.shape == (3, 32, 3) and e < 3e-2, (scale, exact, e)


def test_sync_head_vs_oracle_and_eager(head):
    from oracle import nextdit_sync_oracle as S
    m, sdc, _ = head
    sdb = {k: v.bfloat16() for k, v in sdc.items()}
    B, Ns = 3, 4
    gen = torch.Generator().manual_seed(21)
    lat = torch.randn(B, 4, 3584, generator=gen).cuda()
    x0 = torch.randn(B * Ns, 32, 3, generator=gen).bfloat16().float().cuda()
    for scale in (1.0, 2.5):
        with torch.no_grad():
            t_ref = S.generate_traj(sdc, lat, x0, guidance_scale=scale, num_sample_trajs=Ns)
            t_eag = S.generate_traj(sdb, lat.bfloat16(), x0.bfloat16(), guidance_scale=scale, num_sample_trajs=Ns)
        out = m.generate_traj(lat.bfloat16(), None, guidance_scale=scale, num_sample_trajs=Ns, x_init=x0)
        e, ee = _rel(out, t_ref), _rel(t_eag, t_ref)
        print("sync head, guidance %.1f: rel err" % scale, e, "bf16 eager", ee)
        assert e < 2e-2 and e < 2 * ee + 2e-3, (scale, e, ee)


def test_sync_head_batch_and_graph(head):
    from internnav_b200.internvla_n1 import InternVLAN1ForCausalLM
    m, sdc, _ = head
    B, Ns = 64, 32
    gen = torch.Generator().manual_seed(4)
    lat = torch.randn(B, 4, 3584, generator=gen).bfloat16().cuda()
    x0 = torch.randn(B * Ns, 32, 3, generator=gen).bfloat16().cuda()
    full = m.generate_traj(lat, None, num_sample_trajs=Ns, x_init=x0, guidance_scale=2.0)
    eager = m.generate_traj(lat, None, num_sample_trajs=Ns, x_init=x0, guidance_scale=2.0, graph=False)
    assert torch.equal(full, eager), "the CUDA-graph replay of the sampler differs from the eager launch sequence"
    for b in range(B):
        one = m.generate_traj(lat[b:b + 1], None, num_sample_trajs=Ns, x_init=x0[b * Ns:(b + 1) * Ns], guidance_scale=2.0)
        assert torch.equal(one, full[b * Ns:(b + 1) * Ns]), "environment %d differs in the batch" % b
    # the same head behind the model class, routed from a full state_dict; the frames are ignored
    model = InternVLAN1ForCausalLM(device="cuda:0", system1="nextdit")
    model.model.nextdit.load_state_dict(sdc)
    img = torch.rand(2, 2, 224, 224, 3, device="cuda")
    out = model.generate_traj(lat[:2], img, guidance_scale=2.0, num_sample_trajs=Ns, x_init=x0[:2 * Ns])
    assert torch.equal(out, full[:2 * Ns])
