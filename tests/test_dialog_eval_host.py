"""The batched VL-LN dialog / ObjectNav evaluator (internnav_b200.habitat_dialog) against
tests/golden/habitat_dialog_traces.json, which oracle/gen_golden_dialog.py recorded from the reference's own
`HabitatDialogEvaluator.eval_action` and `DialogAgent`, driven by the scripted simulator, follower, NPC, processor and
model of oracle/habitat_dialog_script.py.  Host frame path (Pillow); CPU only."""
import json
import os
import re

import numpy as np
import pytest
import torch

from oracle import habitat_dialog_script as D
from oracle import habitat_s2_script as S
from oracle import habitat_script as H

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN_PATH = os.path.join(ROOT, "tests", "golden", "habitat_dialog_traces.json")
with open(GOLDEN_PATH, encoding="utf-8") as fh:
    GOLDEN = json.load(fh)
TRACES = GOLDEN["traces"]
MAX_CALLS_ON_ONE_GOAL = 10   # the pixel answer's call, then eight forward steps, then the ninth drops the goal


def _configs():
    """Traces grouped by evaluator configuration (one evaluator serves one task)."""
    out = {}
    for t in TRACES:
        c = t["case"]
        out.setdefault((c["task"], c["dialog_enabled"], c["append_look_down"], c["turn"]), []).append(t)
    return list(out.values())


def _coverage(t):
    from internnav_b200.habitat_dialog import NO_ANSWER, QUESTION_LIMIT
    ev, answers, found, n = t["events"], t["answers"], set(), 0
    for i, e in enumerate(ev):
        if "s2" in e:
            ans = answers[n % len(answers)]
            n += 1
            chat = e["s2"]
            last = chat.rsplit("<|user|>", 1)[1]
            if e["look_down"] and "<image>" in last:
                found.add("look-down turn")
            if e["look_down"] and "<image>" not in last:
                found.add("dialog turn")
            if last.startswith(QUESTION_LIMIT):
                found.add("talk over the limit")
            if last.startswith(NO_ANSWER):
                found.add("NPC answer None")
            if "<|dialog_start|>" in chat:
                found.add("dialog in a later history prompt")
            if "look down image is:<image>" in chat:
                found.add("previous look-down image")
            if "look down image is not here" in chat:
                found.add("no previous look-down image")
            if "<talk>" not in ans and len(re.findall(r"\d+", ans)) == 1:
                found.add("lone number")
        if "npc" in e:
            found.add("talk under the limit")
        if "follow" in e:
            calls = [x.get("follow") for x in ev[:i + 1]]
            prior = calls.count(e["follow"])
            if prior == 1 and e["answer"] == 0:
                found.add("follower 0 at once")
            elif e["answer"] == 0:
                found.add("follower STOP")
            if prior == MAX_CALLS_ON_ONE_GOAL:
                found.add("forward limit")
        if "snap" in e:
            found.add("snapped goal")
    for g in t["geometry"]:
        if g["z"] is None:
            found.add("pixel outside the frame")
    for r in t["results"]:
        if 7 in r["action"]:
            found.add("action 7")
        if r["steps"] == D.MAX_STEPS_PER_EPISODE + 1:
            found.add("step budget")
        elif "error" not in r:
            found.add("done")
        if r.get("error") == "ValueError":
            found.add("continuing a cleared conversation")
    return found


def test_traces_cover_the_loop():
    found = set().union(*(_coverage(t) for t in TRACES))
    assert found == {"look-down turn", "dialog turn", "talk under the limit", "talk over the limit", "NPC answer None",
                     "dialog in a later history prompt", "previous look-down image", "no previous look-down image",
                     "lone number", "pixel outside the frame", "follower 0 at once", "follower STOP", "forward limit",
                     "snapped goal", "action 7", "step budget", "done", "continuing a cleared conversation"}, found
    assert {t["case"]["task"] for t in TRACES} == {"instance_dialog", "objectnav", "coin"}


def test_generator_reproduces_golden_byte_for_byte(tmp_path):
    """`python -m oracle.gen_golden_dialog` rewrites the fixture byte for byte (needs the reference tree)."""
    from oracle.ref_loader import available
    if not available():
        pytest.skip("reference tree not present")
    import oracle.gen_golden_dialog as G
    out = str(tmp_path / "traces.json")
    G.main(out)
    assert open(out, "rb").read() == open(GOLDEN_PATH, "rb").read()


@pytest.mark.parametrize("ti", range(len(TRACES)))
def test_single_environment_reproduces_reference_trace(ti):
    ev = D.replay([TRACES[ti]])
    assert ev.calls["s2"] == sum("s2" in e for e in TRACES[ti]["events"])
    assert ev.calls["npc"] == sum("npc" in e for e in TRACES[ti]["events"])


@pytest.mark.parametrize("ci", range(len(_configs())))
def test_environments_side_by_side_reproduce_their_traces(ci):
    """At most one System-2 call per round, shared by every waiting environment, whatever its turn."""
    traces = _configs()[ci]
    ev = D.replay(traces)
    assert ev.calls["s2"] <= ev.calls["rounds"] and ev.calls["npc"] <= ev.calls["rounds"]
    if len(traces) > 1:
        assert ev.calls["s2"] < sum("s2" in e for t in traces for e in t["events"])


@pytest.mark.parametrize("ci", range(len(_configs())))
def test_environments_rendering_into_one_buffer(ci):
    D.replay(_configs()[ci], reuse_buffer=True)


def test_goals_are_bit_equal_to_the_reference_geometry():
    from internnav_b200 import habitat_eval as HE
    c = GOLDEN["constants"]
    K = HE.intrinsic_matrix(c["width"], c["height"], c["hfov"])
    assert S.reprs(K) == c["intrinsic"]
    geo = [g for t in TRACES for g in t["geometry"]]
    assert geo and any(g["z"] is None for g in geo)
    for g in geo:
        if g["z"] is None:
            continue
        depth = np.zeros((c["height"], c["width"]), dtype=g["z"]["dtype"])
        v, u = g["pixel"]
        depth[v, u] = float(g["z"]["v"])
        tf = np.array([float(x) for x in g["tf"]]).reshape(4, 4)
        assert [repr(float(x)) for x in HE.pixel_to_gps(g["pixel"], depth, K, tf)] == g["out"]


def test_lifted_goals_match_the_follower_calls():
    """Each goal the batched loop lifts is the reference's bit for bit: the replay's follower calls carry the goals as
    exact float64 reprs, and the camera transform of every pixel answer is the reference's."""
    from internnav_b200 import habitat_dialog as HD
    tfs = []
    original = HD.camera_to_episodic

    def logged(xyz, yaw):
        m = original(xyz, yaw)
        tfs.append(S.reprs(m))
        return m
    HD.camera_to_episodic = logged
    try:
        for t in TRACES:
            tfs.clear()
            D.replay([t])
            assert tfs == [g["tf"] for g in t["geometry"]], t["case"]
    finally:
        HD.camera_to_episodic = original


def test_summarize_dialog_equals_calc_metrics():
    from internnav_b200.habitat_dialog import summarize_dialog
    cm = GOLDEN["calc_metrics"]
    inp = cm["inputs"]
    results = [{"success": s, "spl": p, "os": o, "ne": n} for s, p, o, n in
               zip(inp["sucs"], inp["spls"], inp["oss"], inp["nes"])]
    assert summarize_dialog(results) == cm["outputs"]
    got = summarize_dialog([r for t in TRACES for r in t["results"]])
    assert set(got) == {"sucs_all", "spls_all", "oss_all", "nes_all"}


def test_arguments_are_checked():
    from internnav_b200.habitat_dialog import HabitatDialogEvaluator
    model = S.S2Model({}, {})
    kw = dict(depth_filter=H.depth_filter, camera_height=1.25)
    HabitatDialogEvaluator(model, D.Processor({}), **kw)
    with pytest.raises(NotImplementedError):
        HabitatDialogEvaluator(model, D.Processor({}), mode="dual_system", **kw)
    with pytest.raises(ValueError, match="mode"):
        HabitatDialogEvaluator(model, D.Processor({}), mode="system1", **kw)
    with pytest.raises(ValueError, match="camera_height"):
        HabitatDialogEvaluator(model, D.Processor({}), **dict(kw, camera_height=None))
    with pytest.raises(ValueError, match="depth_filter"):
        HabitatDialogEvaluator(model, D.Processor({}), **dict(kw, depth_filter=None))
    with pytest.raises(ValueError, match="generate"):
        HabitatDialogEvaluator(object(), D.Processor({}), **kw)
    with pytest.raises(ValueError, match="npc"):
        HabitatDialogEvaluator(model, D.Processor({}), npc="oracle", **kw)
    ev = D.evaluator(TRACES[:1], {0: []})
    with pytest.raises(ValueError, match="seeds"):
        ev.run([D.DialogEnv(0, 0, 1, []), D.DialogEnv(1, 0, 1, [])])


def test_question_without_npc_ends_only_that_episode():
    """A question in an evaluator without `npc` ends that environment's episode with an error dict."""
    t = next(t for t in TRACES if any("npc" in e for e in t["events"]))
    r = t["case"]["robot"]
    logs = {r: []}
    ev = D.evaluator([t], logs)
    res = ev.run([D.DialogEnv(r, t["case"]["seed"], 1, logs[r], task=t["case"]["task"])])[0]
    assert res[-1]["error"] == "RuntimeError" and "npc" in res[-1]["error_message"]


def test_policy_answers_text_and_keeps_the_base_defaults():
    """DialogPolicy returns the answer text (the loop parses it); the base policy still parses S2Outputs."""
    from internnav_b200 import policy as P
    from internnav_b200.habitat_dialog import DialogPolicy, _Turn
    log = []
    pol = DialogPolicy(S.S2Model({0: ["<talk>where is it?"]}, {0: log}), H.Processor({0: log}), num_envs=1)
    pol.step_no_infer([0], [H.observation(1, 0, 0)["rgb"]])
    out = pol.s2_step([0], [None], [None], [None], [_Turn("fresh", H.instruction(0, 0)[:-1], 0)], None, [False])
    assert out == ["<talk>where is it?"]
    base = P.InternVLAN1Policy(S.S2Model({0: ["240, 320"]}, {0: log}), H.Processor({0: log}), num_envs=1,
                               system2_only=True)
    res = base.s2_step([0], [H.observation(1, 0, 0)["rgb"]], [None], [None], [H.instruction(0, 0)[:-1]], None, [False])
    assert list(res[0].output_pixel) == [320, 240]


def test_kv_capacity_formula():
    from internnav_b200.habitat_dialog import DialogPolicy
    pol = DialogPolicy(S.S2Model({}, {}), H.Processor({}), num_envs=2, num_history=8, resize_w=384, resize_h=384,
                       max_new_tokens=128, turn=5, npc_tokens=128)
    frame, full = 14 * 14, 18 * 23
    assert pol._kv_capacity(480, 640) == (8 + 5 + 2) * frame + full + 7 * 128 + 5 * 128 + 5 * 256 + 512
    assert pol._feature_rows(480, 640) == 2 * ((8 + 5 + 2) * frame + full)
    assert torch.device(pol.device).type == "cpu"
