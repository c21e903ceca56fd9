"""The batched VLN-CE evaluator on the GPU: the device System-1 frames against torch's bf16 division of Pillow's resize,
the device frame path against the reference traces (tests/golden/habitat_eval_traces.json), and a closed loop on the
library's kernels (tiny Qwen2.5-VL config + full-size navdp_async System 1, seeded weights), so that depth is read."""
import json
import os

import numpy as np
import pytest
import torch
from PIL import Image

from oracle import habitat_script as H

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
with open(os.path.join(ROOT, "tests", "golden", "habitat_eval_traces.json"), encoding="utf-8") as fh:
    TRACES = json.load(fh)["traces"]


def _evaluator(device):
    from internnav_b200.habitat_eval import HabitatVLNEvaluator
    model = H.BatchedModel({}, {})
    model.device = torch.device(device)
    return HabitatVLNEvaluator(model, H.Processor({}), depth_filter=H.depth_filter)


def test_shared_s1_rgb_cast_to_bf16_equals_torch_bf16_of_pillow():
    """The evaluator's System-1 RGB: one FramePreprocessor call for all frames (float32 u / 255), cast to bf16 ==
    torch's CPU bf16(Pillow-resized u8) / 255, and == the Pillow path of an evaluator on the CPU."""
    gpu = _evaluator("cuda:0")
    assert gpu._frames is not None
    frames = [H.observation(5, 0, k)["rgb"] for k in range(6)]
    frames.append(np.resize(np.arange(256, dtype=np.uint8), (480, 640, 3)))   # every byte value
    f32 = gpu.s1.rgb(frames)
    assert f32.is_cuda and f32.dtype == torch.float32 and f32.shape == (len(frames), 224, 224, 3)
    got = f32.to(torch.bfloat16)
    want = torch.stack([torch.tensor(np.array(Image.fromarray(f).resize((224, 224)))).to(torch.bfloat16) / 255
                        for f in frames])
    assert torch.equal(got.cpu().view(torch.int16), want.view(torch.int16))
    assert torch.equal(got.cpu().view(torch.int16), _evaluator("cpu").s1.rgb(frames).to(torch.bfloat16).view(torch.int16))


@pytest.mark.parametrize("ti", range(len(TRACES)))
def test_device_frame_path_reproduces_trace(ti):
    ev = H.replay([TRACES[ti]], device="cuda:0")
    assert ev._frames is not None


def test_device_frame_path_side_by_side():
    H.replay(TRACES, device="cuda:0")


def test_device_frame_path_with_environments_rendering_into_one_buffer():
    H.replay(TRACES, device="cuda:0", reuse_buffer=True)


# ------------------------------------------------------------------------------------------------ closed loop
class _Processor:
    """Stand-in for the HF processor with real shapes: characters -> token ids, every image -> a [1, 8, 8] patch grid
    whose pixel rows are seeded by the image's bytes.  `decode` turns the random model's generated ids into a pixel
    goal, look-down, arrows or STOP, chosen by the ids alone, so an environment's answers depend on its own prompt."""

    class _Tok:
        padding_side = "left"

        def decode(self, ids, skip_special_tokens=True):
            ids = [int(i) for i in ids if int(i) < 151643] or [0]
            kind = ids[0] % 7
            if kind < 3:
                return "%d, %d" % (ids[-1] % 480, (ids[0] * 7) % 640)
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


class _Env(H.ScriptedEnv):
    """ScriptedEnv with 96 x 128 frames (cut from the 480 x 640 ones)."""

    def reset(self):
        obs = super().reset()
        return None if obs is None else self._small(obs)

    def step(self, action):
        obs, r, done, info = super().step(action)
        return self._small(obs), r, done, info

    @staticmethod
    def _small(obs):
        return dict(obs, rgb=np.ascontiguousarray(obs["rgb"][::5, ::5]), depth=np.ascontiguousarray(obs["depth"][::5, ::5]))


class _Noise:
    """x_init of the environments an evaluator runs (robots[e] is env e's robot): each robot's n-th System-1 call gets
    its own seeded noise."""

    def __init__(self, robots):
        self.robots, self.n = robots, {r: 0 for r in robots}

    def __call__(self, env_ids):
        out = []
        for e in env_ids:
            r = self.robots[e]
            g = torch.Generator().manual_seed(1000 * r + self.n[r])
            out.append(torch.randn(32, 32, 3, generator=g).to("cuda:0", torch.bfloat16))
            self.n[r] += 1
        return torch.cat(out)


@pytest.fixture(scope="module")
def model():
    from internnav_b200.internvla_n1 import InternVLAN1ForCausalLM
    from internnav_b200.manifest import random_navdp_state_dict
    from oracle import qwen_oracle as Q
    cfg = Q.tiny_cfg()
    m = InternVLAN1ForCausalLM(cfg, device="cuda:0", system1="navdp_async")
    m.load_parts(Q.make_s2_state_dict(cfg, seed=3, lm_head=True), random_navdp_state_dict(5, vlm_token_dim=cfg["hidden"]))
    return m


def _closed_loop(model, robots):
    """Run robots' environments (2 episodes each, 8 steps at most) in one evaluator -> (per robot: results, env log)."""
    from internnav_b200.habitat_eval import HabitatVLNEvaluator
    ev = HabitatVLNEvaluator(model, _Processor(), num_history=4, resize_w=56, resize_h=56, max_steps_per_episode=8,
                             max_new_tokens=6, depth_filter=H.depth_filter, seeds=[40 + r for r in robots],
                             x_init=_Noise(robots))
    logs = {r: [] for r in robots}
    res = ev.run_dual_system([_Env(r, 50 + r, 2, logs[r]) for r in robots])
    out = [({"results": [dict(x, error=type(x["error"]).__name__) if "error" in x else x for x in rs]}, logs[r])
           for r, rs in zip(robots, res)]
    return out, ev


def test_closed_loop_batched_equals_single_environment_drivers(model):
    robots = [0, 1, 2, 3]
    batched, ev = _closed_loop(model, robots)
    again, _ = _closed_loop(model, robots)
    assert batched == again, "two runs differ"
    for j, r in enumerate(robots):
        single, _ = _closed_loop(model, [r])
        assert single[0] == batched[j], "robot %d differs from its single-environment driver" % r
    steps = [e["step"] for _, log in batched for e in log if "step" in e]
    print("calls", ev.calls, "results", [b[0]["results"] for b in batched])
    assert ev.calls["s1"] >= 2 and ev.calls["s2"] >= 2 and ev.reads_depth
    assert set(steps) >= {1, 4, 5} and all(len(b[0]["results"]) == 2 for b in batched)
