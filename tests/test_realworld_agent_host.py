"""The batched real-world agent (internnav_b200/agent_realworld.py) against tests/golden/realworld_agent_traces.json, which
oracle/gen_golden_realworld.py recorded from the reference's own InternVLAN1AsyncAgent driven by the scripted processor
and models of oracle/realworld_script.py.  Host frame path (Pillow); CPU only."""
import json
import os

import numpy as np
import pytest

from oracle import realworld_script as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
with open(os.path.join(ROOT, "tests", "golden", "realworld_agent_traces.json"), encoding="utf-8") as fh:
    TRACES = json.load(fh)["traces"]


def test_traces_cover_the_agent():
    """The fixture exercises every branch of the reference's step: gaps 1 / 4 / 8, resets, look-down retries, pixel
    goals, action answers including an empty one, and an answer the pixel parser rejects."""
    assert {t["case"]["plan_step_gap"] for t in TRACES} == {1, 4, 8}
    frames = [f for t in TRACES for f in t["frames"]]
    assert sum(f["reset"] for f in frames) > len(TRACES)
    assert any(len(f["steps"]) == 2 for f in frames)
    assert any("pixel_goal" in f["result"] for f in frames) and any("error" in f["result"] for f in frames)
    assert any(f["result"].get("discrete_action") == [] for f in frames)
    assert any(len(f["result"].get("discrete_action", [])) > 1 for f in frames)


@pytest.mark.parametrize("ti", range(len(TRACES)))
def test_single_robot_reproduces_reference_trace(ti):
    R.replay_steps(TRACES[ti])


def test_robots_side_by_side_reproduce_their_traces():
    """All traces in one agent (B = number of traces, resets interleaved); a served frame makes at most two System-2
    calls (the due robots, then the look-down retries) and at most one System-1 call."""
    per_frame = []

    def check(agent, before):
        s2, s1 = agent.calls["s2"] - before["s2"], agent.calls["s1"] - before["s1"]
        assert s2 <= 2 and s1 <= 1
        per_frame.append((s2, s1))
    R.replay_serve(TRACES, check_calls=check)
    assert any(s2 == 2 for s2, _ in per_frame) and sum(s1 for _, s1 in per_frame) > 0


def test_waypoints_match_reference_function():
    """Host path of batched_traj_to_waypoints == vln_utils.traj_to_actions(..., use_discrate_action=False) per robot."""
    import torch
    from internnav_b200.postprocess import batched_traj_to_waypoints, traj_to_actions
    t = torch.randn(3 * 5, 7, 3, generator=torch.Generator().manual_seed(1))
    got = batched_traj_to_waypoints(t, 3)
    assert got.dtype == np.float64 and got.shape == (3, 8, 2)
    for b in range(3):
        assert np.array_equal(got[b], traj_to_actions(t[b * 5:(b + 1) * 5].clone(), use_discrate_action=False))


def test_model_without_system1_is_refused():
    from types import SimpleNamespace
    from internnav_b200.agent_realworld import InternVLAN1AsyncAgent
    model = R.ScriptedBatchedModel({0: ["STOP"]}, [])
    model.has_system1 = False
    args = SimpleNamespace(device="cpu", model_path=None, resize_w=384, resize_h=384, num_history=8, plan_step_gap=4)
    with pytest.raises(ValueError, match="System 1"):
        InternVLAN1AsyncAgent(args, model=model, processor=R.ScriptedProcessor([]))
