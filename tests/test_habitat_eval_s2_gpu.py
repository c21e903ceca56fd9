"""The batched VLN-CE evaluator's system2 mode on the GPU: the reference traces (tests/golden/habitat_eval_s2_traces.json)
with the policy on the device, and a closed loop on the library's kernels (tiny Qwen2.5-VL config, seeded weights):
B environments in one driver equal B single-environment drivers byte for byte, and a dual-system model in system2 mode
runs no latent pass and answers as the System-2-only model with the same System-2 weights."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import habitat_s2_script as S
from oracle import habitat_script as H

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
with open(os.path.join(ROOT, "tests", "golden", "habitat_eval_s2_traces.json"), encoding="utf-8") as fh:
    TRACES = json.load(fh)["traces"]


@pytest.mark.parametrize("ti", range(len(TRACES)))
def test_device_policy_reproduces_trace(ti):
    ev = S.replay([TRACES[ti]], device="cuda:0")
    assert ev.policy.device == torch.device("cuda:0")


def test_device_policy_side_by_side_with_one_buffer_environments():
    ev = S.replay(TRACES, device="cuda:0", reuse_buffer=True)
    assert ev.calls["s2"] <= ev.calls["rounds"]


# ------------------------------------------------------------------------------------------------ closed loop
SMALL_H, SMALL_W = 96, 128


class _Processor:
    """Stand-in for the HF processor with real shapes: characters -> token ids, every image -> a [1, 8, 8] patch grid
    whose pixel rows are seeded by the image's bytes.  `decode` turns the random model's generated ids into a pixel
    answer inside the 128 x 96 frame, look-down, arrows or STOP, chosen by the ids alone."""

    class _Tok:
        padding_side = "left"

        def decode(self, ids, skip_special_tokens=True):
            ids = [int(i) for i in ids if int(i) < 151643] or [0]
            kind = ids[0] % 7
            if kind < 3:
                return "%d, %d" % ((ids[0] * 7) % SMALL_W, ids[-1] % SMALL_H)
            if kind == 3:
                return "↓"
            if kind == 4 and ids[-1] % 4 == 0:
                return "STOP"
            return "".join("↑←→"[i % 3] for i in ids[:3])

    def __init__(self):
        self.tokenizer = self._Tok()

    def apply_chat_template(self, conversation, tokenize=False, add_generation_prompt=True):
        return "\n".join(t["role"] + ":" + "".join("<image>" if c["type"] == "image" else c["text"] for c in t["content"])
                         for t in conversation)

    def __call__(self, text, images, return_tensors="pt"):
        ids, rows, grids = [], [], []
        pieces = text[0].split("<image>")
        for i, piece in enumerate(pieces):
            ids += [1000 + (ord(c) % 5000) for c in piece[-48:]]
            if i < len(pieces) - 1:
                seed = int(np.asarray(images[i], dtype=np.int64).sum()) % (2 ** 31)
                rows.append(torch.randn(64, 1176, generator=torch.Generator().manual_seed(seed)))
                grids.append(torch.tensor([1, 8, 8]))
                ids += [151652] + [151655] * 16 + [151653]
        return {"input_ids": torch.tensor([ids]), "pixel_values": torch.cat(rows), "image_grid_thw": torch.stack(grids)}


class _Env(S.ScriptedEnvS2):
    """ScriptedEnvS2 with 96 x 128 frames (cut from the 480 x 640 ones)."""

    def _observe(self):
        obs = super()._observe()
        return dict(obs, rgb=np.ascontiguousarray(obs["rgb"][::5, ::5]), depth=np.ascontiguousarray(obs["depth"][::5, ::5]))


def _tiny(system1):
    from internnav_b200.internvla_n1 import InternVLAN1ForCausalLM
    from internnav_b200.manifest import random_navdp_state_dict
    from oracle import qwen_oracle as Q
    cfg = Q.tiny_cfg()
    m = InternVLAN1ForCausalLM(cfg, device="cuda:0", system1=system1)
    s1 = random_navdp_state_dict(5, vlm_token_dim=cfg["hidden"]) if system1 else None
    m.load_parts(Q.make_s2_state_dict(cfg, seed=3, lm_head=True), s1)
    return m


@pytest.fixture(scope="module")
def s2_model():
    return _tiny(None)


def _closed_loop(model, robots):
    """Run robots' environments (2 episodes each, 10 steps at most) in one system2 evaluator -> (per robot: results and
    env log, the evaluator)."""
    from internnav_b200.habitat_eval import HabitatVLNEvaluator
    ev = HabitatVLNEvaluator(model, _Processor(), mode="system2", num_history=4, resize_w=56, resize_h=56,
                             max_steps_per_episode=10, max_new_tokens=6, depth_filter=H.depth_filter,
                             seeds=[40 + r for r in robots], camera_height=S.CAMERA_HEIGHT, width=SMALL_W,
                             height=SMALL_H, hfov=S.HFOV,
                             make_follower=lambda env: S.ScriptedFollower(env._env.sim, 0.25, False))
    logs = {r: [] for r in robots}
    res = ev.run_system2([_Env(r, 50 + r, 2, logs[r]) for r in robots])
    return [(rs, logs[r]) for r, rs in zip(robots, res)], ev


def test_closed_loop_batched_equals_single_environment_drivers(s2_model):
    robots = [0, 1, 2, 3]
    batched, ev = _closed_loop(s2_model, robots)
    again, _ = _closed_loop(s2_model, robots)
    assert batched == again, "two runs differ"
    for j, r in enumerate(robots):
        single, _ = _closed_loop(s2_model, [r])
        assert single[0] == batched[j], "robot %d differs from its single-environment driver" % r
    events = [e for _, log in batched for e in log]
    print("calls", ev.calls, "results", [b[0] for b in batched])
    assert ev.calls["s2"] >= 2 and ev.calls["s2"] <= ev.calls["rounds"]
    assert any("follow" in e for e in events)   # a pixel answer was lifted and walked
    assert all(len(b[0]) == 2 for b in batched)


def test_dual_system_model_in_system2_mode_runs_no_latent_pass(s2_model):
    dual = _tiny("navdp_async")
    calls = []
    generate_with_latents = dual.generate_with_latents

    def counted(*a, **kw):
        calls.append(1)
        return generate_with_latents(*a, **kw)

    dual.generate_with_latents = counted
    robots = [0, 1, 2]
    got, _ = _closed_loop(dual, robots)
    want, _ = _closed_loop(s2_model, robots)
    assert not calls
    assert got == want
