"""The real-world agent on the GPU: the waypoint kernel (n1_traj_mean_path) against numpy, the device System-1 frame path
against Pillow and the reference traces (tests/golden/realworld_agent_traces.json), and a closed loop on the library's
kernels (tiny Qwen2.5-VL config + full-size nextdit_async head, seeded weights)."""
import json
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch
from PIL import Image

from oracle import realworld_script as R

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
with open(os.path.join(ROOT, "tests", "golden", "realworld_agent_traces.json"), encoding="utf-8") as fh:
    TRACES = json.load(fh)["traces"]


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("T", [8, 24, 32])
@pytest.mark.parametrize("ns", [1, 32])
def test_waypoint_kernel_bit_equal_to_numpy(dtype, T, ns):
    from internnav_b200.postprocess import batched_traj_to_waypoints, traj_to_actions
    g = torch.Generator().manual_seed(T * 100 + ns)
    for B in (1, 5, 64):
        t = (torch.randn(B * ns, T, 3, generator=g) * torch.tensor([0.8, 0.5, 0.1])).to(dtype)
        keep = t.clone()
        got = batched_traj_to_waypoints(t.cuda(), B)
        assert torch.equal(t, keep), "the input was modified"
        assert got.dtype == np.float64 and got.shape == (B, T + 1, 2)
        for b in range(B):
            want = traj_to_actions(t[b * ns:(b + 1) * ns].clone(), use_discrate_action=False)
            assert np.array_equal(got[b], want), (B, b)


def test_shared_s1_frames_equal_pillow():
    """The agent's device frames (one FramePreprocessor call per step) hold the bytes of the reference's Pillow resize:
    RGB x / 255 exactly as float32, depth in mode F with no scaling or clip."""
    gpu, cpu = R.make_agent(TRACES[:1], "cuda:0")[0], R.make_agent(TRACES[:1], "cpu")[0]
    obs = [R.frame(5, k) for k in range(6)]
    rgb_gpu = gpu.s1.rgb([o[0] for o in obs])
    assert rgb_gpu.is_cuda and rgb_gpu.dtype == torch.float32
    assert torch.equal(rgb_gpu.cpu(), cpu.s1.rgb([o[0] for o in obs]))
    pil = np.stack([np.array(Image.fromarray(o[0]).resize((224, 224))) / 255 for o in obs])   # the reference, float64
    assert torch.equal(rgb_gpu.cpu(), torch.from_numpy(pil).float())
    dep_gpu = gpu.s1.depth([o[1] for o in obs])
    pil_d = np.stack([np.array(Image.fromarray(o[1]).resize((224, 224))) for o in obs])
    assert torch.equal(dep_gpu.cpu(), torch.from_numpy(pil_d)) and float(pil_d.max()) > 5.0   # no clip


@pytest.mark.parametrize("ti", range(len(TRACES)))
def test_device_frame_path_reproduces_trace(ti):
    agent = R.replay_steps(TRACES[ti], device="cuda:0")
    assert agent._frames is not None


def test_device_frame_path_serves_traces_side_by_side():
    R.replay_serve(TRACES, device="cuda:0")


# ------------------------------------------------------------------------------------------------ closed loop
class _Processor:
    """Stand-in for the HF processor with real shapes: characters -> token ids, every image -> a [1, 8, 8] patch grid
    whose pixel rows are seeded by the image's bytes.  `decode` turns the generated ids of the random model into an
    answer chosen by the ids alone (a pixel goal, arrows or look-down), so a robot's answers depend on its own prompt."""

    class _Tok:
        padding_side = "left"

        def decode(self, ids, skip_special_tokens=True):
            ids = [int(i) for i in ids if int(i) < 151643] or [0]
            kind = ids[0] % 5
            if kind < 3:
                return "%d, %d" % (ids[-1] % 480, (ids[0] * 7) % 640)
            return "↓" if kind == 3 else "".join("↑←→"[i % 3] for i in ids[:3])

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


def _noise(robot, n):
    g = torch.Generator().manual_seed(1000 * robot + n)
    return torch.randn(32, 32, 3, generator=g).to("cuda:0", torch.bfloat16)


class _Noise:
    """x_init of the robots an agent serves (robots[e] is env e's robot): each robot's n-th System-1 call gets _noise."""

    def __init__(self, robots):
        self.robots, self.n = robots, {r: 0 for r in robots}

    def __call__(self, env_ids):
        out = []
        for e in env_ids:
            r = self.robots[e]
            out.append(_noise(r, self.n[r]))
            self.n[r] += 1
        return torch.cat(out)


@pytest.fixture(scope="module")
def model():
    from internnav_b200.internvla_n1 import InternVLAN1ForCausalLM
    from internnav_b200.manifest import random_nextdit_state_dict
    from oracle import qwen_oracle as Q
    cfg = Q.tiny_cfg()
    m = InternVLAN1ForCausalLM(cfg, device="cuda:0", system1="nextdit_async")
    m.load_parts(Q.make_s2_state_dict(cfg, seed=3, lm_head=True), random_nextdit_state_dict(5, vlm_token_dim=cfg["hidden"]))
    return m


def _closed_loop(model, robots, frames=8):
    """Serve `robots` in one agent, frames of 96 x 128, robot 3 starting a new episode at frame 5 -> per frame the list
    of results (and the agent)."""
    from internnav_b200.agent_realworld import InternVLAN1AsyncAgent
    args = SimpleNamespace(device="cuda:0", model_path=None, resize_w=56, resize_h=56, num_history=4, plan_step_gap=2)
    agent = InternVLAN1AsyncAgent(args, model=model, processor=_Processor(), num_envs=len(robots), x_init=_Noise(robots))
    agent.policy.max_new_tokens = 6
    out = []
    for k in range(frames):
        obs = [R.frame(r, k) for r in robots]
        rgbs = [np.ascontiguousarray(o[0][::5, ::5][:96, :128]) for o in obs]
        depths = [np.ascontiguousarray(o[1][::5, ::5][:96, :128]) for o in obs]
        res = agent.serve(list(range(len(robots))), rgbs, depths, ["walk to door %d" % r for r in robots],
                          resets=[k == 0 or (k == 5 and r == 3) for r in robots])
        out.append([{"error": type(x).__name__} if isinstance(x, Exception) else x for x in res])
    return out, agent


def test_closed_loop_batched_equals_single_robot_agents(model):
    robots = [0, 1, 2, 3]
    batched, agent = _closed_loop(model, robots)
    again, _ = _closed_loop(model, robots)
    assert batched == again, "two runs differ"
    singles = [_closed_loop(model, [r])[0] for r in robots]
    for j, r in enumerate(robots):
        assert [f[j] for f in batched] == [f[0] for f in singles[j]], "robot %d differs from its single-robot agent" % r
    flat = [x for f in batched for x in f]
    trajs = [x for x in flat if "trajectory" in x]
    print("calls", agent.calls, "results", [sorted(x) for x in flat])
    assert trajs and all(np.isfinite(np.asarray(x["trajectory"])).all() and len(x["trajectory"]) == 33 for x in trajs)
    assert agent.calls["s1"] >= 2 and agent.calls["s2"] >= 2
