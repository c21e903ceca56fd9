"""The batched VLN-CE evaluator's system2 mode (HabitatVLNEvaluator.run_system2) against
tests/golden/habitat_eval_s2_traces.json, which oracle/gen_golden_habitat_s2.py recorded from the reference's own
`_run_eval_system2` driven by the scripted simulator, follower, processor and model of oracle/habitat_s2_script.py.
Host frame path (Pillow); CPU only."""
import json
import os
import re

import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

from oracle import habitat_s2_script as S
from oracle import habitat_script as H

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN_PATH = os.path.join(ROOT, "tests", "golden", "habitat_eval_s2_traces.json")
with open(GOLDEN_PATH, encoding="utf-8") as fh:
    GOLDEN = json.load(fh)
TRACES = GOLDEN["traces"]


def _coverage(t):
    ev, answers, found, n = t["events"], t["answers"], set(), 0
    for i, e in enumerate(ev):
        if "s2" in e:
            ans = answers[n % len(answers)]
            n += 1
            if e["look_down"]:
                found.add("look-down turn")
            if len(re.findall(r"\d+", ans)) >= 2:
                found.add("pixel on look-down turn" if e["look_down"] else "pixel on fresh turn")
            for name, pat in [("action answer", "[↑←→]+"), ("look-down alone", "↓"), ("look-down then arrows", "↓[↑←→]+"),
                              ("stop answer", "STOP")]:
                if re.fullmatch(pat, ans):
                    found.add(name)
        if "depth" in e:
            fol = [ev[j] for j in range(i + 1, len(ev)) if "follow" in ev[j]][:2]
            if fol and fol[0]["answer"] == 0:
                found.add("follower STOP at once")
            elif len(fol) == 2 and fol[1]["answer"] == 0 and fol[1]["follow"] == fol[0]["follow"]:
                found.add("follower STOP on second call")
        if "follow" in e:
            found.add("follower returns " + e["as"])
            same = sum(x.get("follow") == e["follow"] for x in ev[:i + 1])
            if same == MAX_CALLS_ON_ONE_GOAL:
                found.add("forward limit")
        if "snap" in e:
            found.add("snapped goal")
    for r in t["results"]:
        if r["steps"] == S.MAX_STEPS_PER_EPISODE + 1:
            found.add("step budget")
        elif "error" not in r:
            found.add("done")
        if r.get("error") == "IndexError":
            found.add("pixel outside the frame" if "out of bounds" in r["error_message"] else "lone number")
        if r.get("error") == "ValueError":
            found.add("look-down after arrows")
    return found


MAX_CALLS_ON_ONE_GOAL = 10   # the pixel-goal iteration's two calls, then eight forward steps, then the ninth drops it


def test_traces_cover_the_loop():
    found = set().union(*(_coverage(t) for t in TRACES))
    assert found == {"look-down turn", "pixel on look-down turn", "pixel on fresh turn", "action answer",
                     "look-down alone", "look-down then arrows", "stop answer", "follower STOP at once",
                     "follower STOP on second call", "follower returns tensor", "follower returns array",
                     "follower returns int", "forward limit", "snapped goal", "step budget", "done",
                     "pixel outside the frame", "lone number", "look-down after arrows"}, found


def test_generator_reproduces_golden_byte_for_byte(tmp_path):
    """`python -m oracle.gen_golden_habitat_s2` rewrites the fixture byte for byte (needs the reference tree)."""
    from oracle.ref_loader import available
    if not available():
        pytest.skip("reference tree not present")
    import oracle.gen_golden_habitat_s2 as G
    out = str(tmp_path / "traces.json")
    G.main(out)
    assert open(out, "rb").read() == open(GOLDEN_PATH, "rb").read()


@pytest.mark.parametrize("ti", range(len(TRACES)))
def test_single_environment_reproduces_reference_trace(ti):
    ev = S.replay([TRACES[ti]])
    assert ev.calls["s2"] == sum("s2" in e for e in TRACES[ti]["events"]) and ev.calls["s1"] == 0


def test_environments_side_by_side_reproduce_their_traces():
    """At most one System-2 call per round, shared by every waiting environment."""
    ev = S.replay(TRACES)
    assert ev.calls["s2"] <= ev.calls["rounds"]
    assert ev.calls["s2"] < sum("s2" in e for t in TRACES for e in t["events"])


@pytest.mark.parametrize("ti", range(len(TRACES)))
def test_environment_rendering_into_one_buffer_reproduces_trace(ti):
    S.replay([TRACES[ti]], reuse_buffer=True)


def test_environments_rendering_into_one_buffer_side_by_side():
    S.replay(TRACES, reuse_buffer=True)


def test_depth_is_filtered_only_for_pixel_answers():
    """The reference filters every frame; the evaluator filters only the frames it lifts a pixel answer on, and the
    goals (hence every follower call in the replay) are the same."""
    calls = []

    def counting(depth, blur_type=None):
        calls.append(depth.shape)
        return H.depth_filter(depth, blur_type=blur_type)

    S.replay(TRACES, depth_filter=counting)
    lifted = sum("depth" in e for t in TRACES for e in t["events"])
    assert len(calls) == lifted and all(s == (H.HEIGHT, H.WIDTH) for s in calls)
    assert sum(t["reference_filter_calls"] for t in TRACES) > 3 * lifted


def test_geometry_is_bit_equal_to_the_reference():
    from internnav_b200 import habitat_eval as HE
    c = GOLDEN["constants"]
    K = HE.intrinsic_matrix(c["width"], c["height"], c["hfov"])
    assert S.reprs(K) == c["intrinsic"] and HE.AXIS_ALIGN.tolist() == c["axis_align"]
    geo = [g for t in TRACES for g in t["geometry"]]
    assert len(geo) == sum("depth" in e for t in TRACES for e in t["events"])
    for g in geo:
        q = [float(v) for v in g["quat"]]
        assert S.reprs(HE.rotation_matrix(q)) == g["rot"]
        xyz = np.array([float(v) for v in g["xyz"]["v"]], dtype=g["xyz"]["dtype"])
        yaw = np.dtype(g["yaw"]["dtype"]).type(float(g["yaw"]["v"]))
        assert g["pitch"] == repr(float(HE.CAMERA_PITCH))
        tf = HE.camera_to_episodic(xyz, yaw)
        assert S.reprs(tf) == g["tf"]
        if g["z"] is None:
            continue
        depth = np.zeros((c["height"], c["width"]), dtype=g["z"]["dtype"])
        v, u = g["pixel"]
        depth[v, u] = float(g["z"]["v"])
        assert [repr(float(x)) for x in HE.pixel_to_gps(g["pixel"], depth, K, tf)] == g["out"]


def test_rotation_matrix_matches_scipy():
    """numpy-quaternion's scalar-first conversion == scipy's (scalar-last input) on unit quaternions, to rounding."""
    from internnav_b200.habitat_eval import rotation_matrix
    rng = np.random.Generator(np.random.PCG64(3))
    for _ in range(200):
        q = rng.normal(size=4)
        q /= np.linalg.norm(q)
        want = Rotation.from_quat([q[1], q[2], q[3], q[0]]).as_matrix()
        np.testing.assert_allclose(rotation_matrix(q), want, rtol=0, atol=2e-15)
        np.testing.assert_allclose(rotation_matrix(S.Quat(*q)), want, rtol=0, atol=2e-15)
    np.testing.assert_array_equal(rotation_matrix([2.0, 0.0, 0.0, 0.0]), np.eye(3))


@pytest.mark.parametrize("value,want", [(torch.tensor([3]), 3), (np.array([2]), 2), (1, 1), (np.int64(0), 0)])
def test_follower_answers_are_normalised(value, want):
    from internnav_b200.habitat_eval import follower_action
    assert follower_action(value) == want


def test_dual_system_model_runs_no_latent_pass():
    """In system2 mode the policy calls generate alone, whatever the model carries; the traces are the same."""
    logs = {t["case"]["robot"]: [] for t in TRACES}
    model = S.S2Model({t["case"]["robot"]: t["answers"] for t in TRACES}, logs)
    model.has_system1 = True
    model.config = H.BatchedModel.config
    S.replay(TRACES, model=model)
    assert model.latent_calls == 0


def test_policy_default_still_computes_latent_plans():
    from internnav_b200 import policy as P
    log = []
    model = H.BatchedModel({0: ["240, 320"]}, {0: log})
    pol = P.InternVLAN1Policy(model, H.Processor({0: log}), num_envs=1)
    res = pol.s2_step([0], [H.observation(1, 0, 0)["rgb"]], [None], [None], [H.instruction(0, 0)[:-1]], None, [False])
    assert pol.latent_plans and res[0].output_latent is not None
    pol = P.InternVLAN1Policy(S.S2Model({0: ["240, 320"]}, {0: log}), H.Processor({0: log}), num_envs=1,
                              system2_only=True)
    res = pol.s2_step([0], [H.observation(1, 0, 0)["rgb"]], [None], [None], [H.instruction(0, 0)[:-1]], None, [False])
    assert not pol.latent_plans and res[0].output_latent is None and list(res[0].output_pixel) == [320, 240]


def test_modes_are_refused_by_the_other_run():
    from internnav_b200.habitat_eval import HabitatVLNEvaluator
    dual = HabitatVLNEvaluator(H.BatchedModel({}, {}), H.Processor({}), depth_filter=H.depth_filter)
    with pytest.raises(ValueError, match="mode='system2'"):
        dual.run_system2([S.ScriptedEnvS2(0, 0, 1, [])])
    s2 = S.evaluator(TRACES[:1], {0: []}, depth_filter=H.depth_filter)
    with pytest.raises(ValueError, match="mode='dual_system'"):
        s2.run_dual_system([H.ScriptedEnv(0, 0, 1, [])])


def test_system2_mode_arguments_are_checked():
    from internnav_b200.habitat_eval import HabitatVLNEvaluator
    model = S.S2Model({}, {})
    kw = dict(mode="system2", depth_filter=H.depth_filter, camera_height=1.25)
    HabitatVLNEvaluator(model, H.Processor({}), **kw)            # a System-2-only model is accepted
    with pytest.raises(ValueError, match="camera_height"):
        HabitatVLNEvaluator(model, H.Processor({}), **dict(kw, camera_height=None))
    with pytest.raises(ValueError, match="depth_filter"):
        HabitatVLNEvaluator(model, H.Processor({}), **dict(kw, depth_filter=None))
    with pytest.raises(ValueError, match="mode"):
        HabitatVLNEvaluator(model, H.Processor({}), **dict(kw, mode="system1"))
    with pytest.raises(ValueError, match="generate"):
        HabitatVLNEvaluator(object(), H.Processor({}), **kw)
