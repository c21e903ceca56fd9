"""The System-1 configurations the reference builds from config.system1 (internvla_n1_arch.py L121-145) -- CPU only.

  * no `system1`: System 2 alone (no latent_queries, no trajectory head),
  * "nextdit": the synchronous DiT head (no RGB branch),
  * "navdp": refused (the reference builds no navdp module for it).

config.json is read in both layouts (flat transformers 4.51, nested 5.x).  The library-backed pieces are stubbed: System 2
records what it is given, and the NextDiT head runs its real load_state_dict on the CPU, whose missing-key check is the
strict load.  The synchronous oracle (oracle/nextdit_sync_oracle.py) is pinned to the reference's own generate_traj run
(tests/golden/nextdit_sync_reference.npz, recorded by `python -m oracle.gen_golden_nextdit_sync`) and, where the reference
tree exists, to the reference classes live."""
import json
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from internnav_b200 import internvla_n1 as M
from internnav_b200 import nextdit
from internnav_b200.manifest import nextdit_shapes, random_nextdit_state_dict

GOLD = os.path.join(os.path.dirname(__file__), "golden", "nextdit_sync_reference.npz")
FLAT = dict(architectures=["InternVLAN1ForCausalLM"], model_type="internvla_n1", hidden_size=256, num_hidden_layers=2,
            num_attention_heads=2, num_key_value_heads=1, intermediate_size=512, vocab_size=1024, rms_norm_eps=1e-6,
            rope_theta=1000000.0, rope_scaling={"type": "mrope", "mrope_section": [16, 24, 24]}, n_query=4)


def _nested(conf):
    out = {k: v for k, v in conf.items() if k in ("n_query", "system1", "architectures", "model_type")}
    out["text_config"] = {k: v for k, v in conf.items() if k not in out}
    return out


def _rel(a, b):
    a, b = torch.as_tensor(a).float(), torch.as_tensor(b).float()
    return float((a - b).norm() / (b.norm() + 1e-12))


class _FakeS2:
    def __init__(self, cfg, device="cuda:0"):
        self.cfg, self.device, self.keys = cfg, torch.device(device), None

    def load_state_dict(self, sd):
        self.keys = set(sd)


class _CpuHead(nextdit.NextDiTSystem1):
    """The NextDiT head with its real load_state_dict, constructed without a device."""

    def __init__(self, device="cuda:0", num_inference_steps=10, asynchronous=True):
        self.device, self.asynchronous, self.num_inference_steps, self.w = torch.device("cpu"), asynchronous, 10, None

    def load_state_dict(self, sd):
        self.keys = set(sd)
        return super().load_state_dict(sd)


@pytest.fixture
def stubbed(monkeypatch):
    monkeypatch.setattr(M, "System2", _FakeS2)
    monkeypatch.setattr(nextdit, "NextDiTSystem1", _CpuHead)


S2_KEYS = {"visual.patch_embed.proj.weight": torch.zeros(4, 4), "model.embed_tokens.weight": torch.zeros(8, 4),
           "model.norm.weight": torch.ones(4), "lm_head.weight": torch.zeros(8, 4)}


def _write(path, conf, sd):
    from safetensors.torch import save_file
    path.mkdir()
    save_file({k: v.contiguous() for k, v in sd.items()}, str(path / "model.safetensors"))
    (path / "config.json").write_text(json.dumps(conf))
    return str(path)


@pytest.mark.parametrize("layout", ["flat", "nested"])
def test_checkpoint_without_system1_is_system2_only(tmp_path, stubbed, layout):
    conf = FLAT if layout == "flat" else _nested(FLAT)
    assert "system1" not in conf
    m = M.InternVLAN1ForCausalLM.from_pretrained(_write(tmp_path / "ck", conf, S2_KEYS), device_map={"": "cuda:0"})
    assert m.get_system1_type() is None and not m.has_system1
    assert m.model.navdp is None and m.model.nextdit is None
    assert m._s2.keys == set(S2_KEYS) and m._s2.cfg["hidden"] == 256
    lat = torch.zeros(1, 4, 256)
    for call in (lambda: m.generate_latents([[1, 2]], None, []), lambda: m.generate_traj(lat, None),
                 lambda: m.generate_with_latents([[1, 2]], None, []), lambda: m.generate([[1, 2]], None, [], with_latents=True),
                 lambda: m.forward(input_ids=[[1]], labels=[[1]], t_s_pos=[0], traj_images=torch.zeros(1)),
                 lambda: m.dual_system_step([[1, 2]], None, [], None, None)):
        with pytest.raises(RuntimeError, match="System 1"):
            call()
    with pytest.raises(ValueError):
        m.load_parts(S2_KEYS, {"x": torch.zeros(1)})
    assert M.Qwen2_5_VLForConditionalGeneration is M.InternVLAN1ForCausalLM


@pytest.mark.parametrize("layout", ["flat", "nested"])
def test_nextdit_checkpoint_routes_the_synchronous_head(tmp_path, stubbed, layout):
    conf = dict(FLAT, system1="nextdit")
    conf = conf if layout == "flat" else _nested(conf)
    head = random_nextdit_state_dict(1, dtype=torch.bfloat16, asynchronous=False)
    sd = dict(S2_KEYS, **{"model.latent_queries": torch.zeros(1, 4, 4)}, **{"model." + k: v for k, v in head.items()})
    m = M.InternVLAN1ForCausalLM.from_pretrained(_write(tmp_path / "ck", conf, sd), device_map={"": "cuda:0"})
    assert m.get_system1_type() == "nextdit" and m.model.navdp is None and not m.model.nextdit.asynchronous
    assert m.model.nextdit.keys == set(nextdit_shapes(asynchronous=False)) == set(head)
    assert m._s2.keys == set(S2_KEYS) | {"model.latent_queries"}
    assert m.model.nextdit.w["dit.kv.w"].shape == (12 * 768, 384) and "vit.patch.w" not in m.model.nextdit.w
    # strict: a head tensor missing from the checkpoint is an error
    m2 = M.InternVLAN1ForCausalLM(m.cfg, system1="nextdit")
    with pytest.raises(KeyError):
        m2.load_state_dict({k: v for k, v in sd.items() if k != "model.traj_dit.model.layers.3.gate"})


def test_asynchronous_head_keeps_its_rgb_branch(stubbed):
    m = M.InternVLAN1ForCausalLM(dict(M.QWEN25VL_7B), system1="nextdit_async")
    head = random_nextdit_state_dict(2, dtype=torch.bfloat16)
    m.load_state_dict(dict(S2_KEYS, **{"model." + k: v for k, v in head.items()}))
    assert m.model.nextdit.asynchronous and m.model.nextdit.keys == set(head) and m._s2.keys == set(S2_KEYS)
    assert "vit.patch.w" in m.model.nextdit.w


@pytest.mark.parametrize("layout", ["flat", "nested"])
def test_navdp_without_async_is_refused(tmp_path, stubbed, layout):
    conf = dict(FLAT, system1="navdp")
    conf = conf if layout == "flat" else _nested(conf)
    with pytest.raises(NotImplementedError, match="navdp"):
        M.InternVLAN1ForCausalLM.from_pretrained(_write(tmp_path / "ck", conf, S2_KEYS), device_map={"": "cuda:0"})


def test_policy_and_registry_without_system1(stubbed):
    from internnav_b200 import registry
    from oracle import policy_script
    model = M.InternVLAN1ForCausalLM(dict(M.QWEN25VL_7B), system1=None)
    conf = registry.InternVLAN1ModelConfig(model_cfg={"model": dict(model_path="unused", device="cpu")})
    net = registry.InternVLAN1Net(conf, model=model, processor=policy_script.FakeProcessor())
    assert net.model_config.system1 is None and not net.has_system1
    with pytest.raises(RuntimeError, match="System 1"):
        net.s1_step_latent([0], [torch.zeros(1, 2, 224, 224, 3)], [torch.zeros(1, 2, 224, 224, 1)],
                           [torch.zeros(1, 4, 3584)])
    bad = registry.InternVLAN1ModelConfig(model_cfg={"model": dict(model_path="unused", device="cpu", system1="nextdit")})
    with pytest.raises(ValueError, match="system1"):
        registry.InternVLAN1Net(bad, model=model, processor=policy_script.FakeProcessor())


def test_oracle_sync_branch_matches_the_reference_run():
    from oracle import nextdit_sync_oracle as S
    from oracle.gen_golden_nextdit import make_inputs
    g = np.load(GOLD)
    sd = random_nextdit_state_dict(int(g["seed"]), asynchronous=False)
    inp = make_inputs(int(g["seed"]), int(g["batch"]), int(g["ns"]))
    with torch.no_grad():
        cond = S.condition_tokens(sd, inp["traj_latents"])
        assert cond.shape == (1, 4, 768) and _rel(cond, g["condition_tokens"]) < 2e-5
        for scale, key in ((1.0, "traj_scale_1"), (2.5, "traj_scale_2p5")):
            out = S.generate_traj(sd, inp["traj_latents"], inp["x_init"], guidance_scale=scale,
                                  num_sample_trajs=int(g["ns"]))
            assert out.shape == (3, 32, 3)
            assert _rel(out, g[key]) < 5e-5, (scale, _rel(out, g[key]))
    assert _rel(g["traj_scale_1"], g["traj_scale_2p5"]) > 1e-3


def test_state_dict_keys_and_sampler_against_the_reference_classes():
    from oracle import ref_loader
    if not ref_loader.available():
        pytest.skip("reference tree not present")
    from oracle import nextdit_sync_oracle as S
    from oracle.gen_golden_nextdit_sync import build_reference_sync_model, reference_meta_model
    ref = {k for k in reference_meta_model("nextdit").state_dict() if "freqs_cis" not in k}
    assert ref == set(nextdit_shapes(asynchronous=False)) | {"latent_queries"}
    assert not reference_meta_model(None).state_dict()           # no system1: no latent_queries, no head
    sd = random_nextdit_state_dict(7, asynchronous=False)
    mod, generate_traj, self_, _ = build_reference_sync_model(sd)
    gen = torch.Generator().manual_seed(11)
    lat, x0 = torch.randn(1, 4, 3584, generator=gen), torch.randn(2, 32, 3, generator=gen)
    mod.randn_tensor = lambda shape, generator=None, device=None, dtype=None: x0.to(dtype).clone()
    with torch.no_grad():
        ref_out = generate_traj(self_, lat, None, guidance_scale=3.0, num_sample_trajs=2)
        mine = S.generate_traj(sd, lat, x0, guidance_scale=3.0, num_sample_trajs=2)
    assert _rel(mine, ref_out) < 5e-5
