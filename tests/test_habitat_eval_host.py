"""The batched VLN-CE evaluator (internnav_b200/habitat_eval.py) against tests/golden/habitat_eval_traces.json, which
oracle/gen_golden_habitat.py recorded from the reference's own `_run_eval_dual_system` driven by the scripted simulator,
processor and models of oracle/habitat_script.py.  Host frame path (Pillow); CPU only."""
import json
import math
import os
import warnings
from collections import Counter

import numpy as np
import pytest
import torch
from PIL import Image

from oracle import habitat_script as H

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
with open(os.path.join(ROOT, "tests", "golden", "habitat_eval_traces.json"), encoding="utf-8") as fh:
    GOLDEN = json.load(fh)
TRACES = GOLDEN["traces"]


def _chunk(ev):
    """The local action chunk the loop takes from one recorded System-1 call (padded to 8, cut to 4)."""
    from internnav_b200.postprocess import traj_to_actions
    ids = traj_to_actions(H.trajectory(ev["s1"], ev["rgb"], ev["depth"]))
    return (ids + [0] * 8)[:4]


def _coverage(trace):
    ev, robot = trace["events"], trace["case"]["robot"]
    answers, n_s2, seen = trace["answers"], 0, Counter()
    found = set()
    for i, e in enumerate(ev):
        nxt = ev[i + 1] if i + 1 < len(ev) else {}
        if "s2" in e:
            ans = answers[n_s2 % len(answers)]
            n_s2 += 1
            found.add("look-down turn") if e["look_down"] else None
            if ans == "STOP" and nxt == {"step": 0}:
                found.add("stop answer")
            if ans and set(ans) <= set("↑←→"):
                found.add("action answer")
            # a re-ask without an environment step: two look-down views in a row before this call (System-1 calls
            # take no step)
            if [x.get("step") for x in ev[:i] if "s1" not in x][-8:] == [5, 5, 4, 4] * 2:
                last = next(x for x in reversed(ev[:i]) if "s1" in x)
                found.add("forward > 8" if seen[last["s1"]] >= 3 else "later local 0")
        if "s1" in e:
            assert e["s1"] // 1000 == robot
            seen[e["s1"]] += 1
            if seen[e["s1"]] == 2:
                found.add("system 1 re-run")
            if seen[e["s1"]] == 1 and _chunk(e)[0] == 0 and nxt == {"step": 2}:
                found.add("first id 0 -> LEFT")
        if [x.get("step") for x in ev[i:i + 4]] == [5, 5, 5, 5]:
            found.add("double look-down")
    if len(trace["results"]) > 1:
        found.add("several episodes")
    if any(r["steps"] == H.MAX_STEPS_PER_EPISODE + 1 for r in trace["results"]):
        found.add("step budget")
    if any("error" in r for r in trace["results"]):
        found.add("raising answer")
    return found


def test_traces_cover_the_loop():
    """Every branch of the reference loop occurs in the fixture."""
    found = set().union(*(_coverage(t) for t in TRACES))
    assert found == {"action answer", "look-down turn", "double look-down", "system 1 re-run", "forward > 8",
                     "first id 0 -> LEFT", "later local 0", "stop answer", "step budget", "raising answer",
                     "several episodes"}, found


@pytest.mark.parametrize("ti", range(len(TRACES)))
def test_single_environment_reproduces_reference_trace(ti):
    ev = H.replay([TRACES[ti]])
    assert ev.calls["s2"] + ev.calls["s1"] == sum("s2" in e or "s1" in e for e in TRACES[ti]["events"])


def test_environments_side_by_side_reproduce_their_traces():
    """All traces in one evaluator: each round makes at most one System-2 and one System-1 call, so the calls are
    batched across environments."""
    ev = H.replay(TRACES)
    requests = {k: sum(k in e for t in TRACES for e in t["events"]) for k in ("s2", "s1")}
    assert ev.calls["s2"] <= ev.calls["rounds"] and ev.calls["s1"] <= ev.calls["rounds"]
    assert ev.calls["s2"] < requests["s2"] and ev.calls["s1"] < requests["s1"]


@pytest.mark.parametrize("ti", range(len(TRACES)))
def test_environment_rendering_into_one_buffer_reproduces_trace(ti):
    """A simulator may write every observation into the same arrays; the reference copies each frame before its next
    step (and its trace is the same either way, which the fixture generator checks), so the evaluator must too."""
    H.replay([TRACES[ti]], reuse_buffer=True)


def test_environments_rendering_into_one_buffer_side_by_side():
    H.replay(TRACES, reuse_buffer=True)


def test_episode_dicts_are_json_serialisable():
    """Every returned dict can be written as the reference writes progress.json, the failed answer's included."""
    from internnav_b200.habitat_eval import HabitatVLNEvaluator
    t = next(t for t in TRACES if any("error" in r for r in t["results"]))
    log = []
    ev = HabitatVLNEvaluator(H.BatchedModel({t["case"]["robot"]: t["answers"]}, {t["case"]["robot"]: log}),
                             H.Processor({t["case"]["robot"]: log}), max_steps_per_episode=H.MAX_STEPS_PER_EPISODE,
                             depth_filter=H.depth_filter, seeds=[t["case"]["seed"]])
    res = ev.run_dual_system([H.ScriptedEnv(t["case"]["robot"], t["case"]["seed"], t["episodes_run"], log)])[0]
    failed = [r for r in res if "error" in r]
    assert failed and failed[0]["error"] == "IndexError" and failed[0]["error_message"]
    assert json.loads(json.dumps(res)) == res


@pytest.mark.parametrize("n_seeds", [1, 3])
def test_seeds_must_match_environments(n_seeds):
    from internnav_b200.habitat_eval import HabitatVLNEvaluator
    ev = HabitatVLNEvaluator(H.BatchedModel({}, {}), H.Processor({}), depth_filter=H.depth_filter,
                             seeds=list(range(n_seeds)))
    with pytest.raises(ValueError, match="seeds"):
        ev.run_dual_system([H.ScriptedEnv(r, r, 1, []) for r in range(2)])


@pytest.mark.parametrize("n_out", [224, 1, 3, 7, 100, 384, 641])
def test_nearest_index_equals_pillow(n_out):
    """nearest_index is the source pixel of Pillow's I;16 NEAREST resize, for every input size up to 1100 and some
    camera sizes (a row of indices as the image)."""
    from internnav_b200.habitat_eval import nearest_index
    for n_in in list(range(1, 1100)) + [1280, 1440, 1920, 2048, 4000]:
        row = np.arange(n_in, dtype=np.uint16)[None, :].repeat(2, axis=0)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", DeprecationWarning)
            img = Image.fromarray(row, mode="I;16")
        got = np.array(img.resize((n_out, 2), Image.NEAREST))[0].astype(np.int64)
        assert np.array_equal(got, nearest_index(n_in, n_out)), (n_in, n_out)


@pytest.mark.parametrize("shape,lo,hi", [((480, 640), 0.0, 10.0), ((256, 320), 0.5, 5.0), ((480, 640, 1), 0.1, 20.0),
                                          ((333, 517), 0.0, 10.0)])
def test_host_depth_equals_full_frame_path(shape, lo, hi):
    """s1_depth == the reference's full-frame path: filter, affine, * 1000, uint16, Pillow I;16 NEAREST to 224 x 224
    (preprocess_depth_image_v2), / 1000, float32, clip at 5, bf16 -- bit for bit, including values on and just below
    integers after * 1000."""
    from internnav_b200.habitat_eval import HabitatVLNEvaluator
    ev = HabitatVLNEvaluator(H.BatchedModel({}, {}), H.Processor({}), min_depth=lo, max_depth=hi,
                             depth_filter=H.depth_filter)
    for k in range(3):
        raw = H.observation(k, 0, 0)["depth"][:, :, 0]
        raw = np.ascontiguousarray(raw[:shape[0], :shape[1]]).reshape(shape)
        d = H.depth_filter(raw.reshape(raw.shape[:2]), blur_type=None)
        d = d * (hi - lo) + lo
        d = d * 1000
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", DeprecationWarning)
            img = Image.fromarray(d.astype(np.uint16), mode="I;16")
        ref = np.array(img.resize((224, 224), Image.NEAREST)) / 1000
        ref = torch.as_tensor(np.ascontiguousarray(ref)).float()
        ref[ref > 5.0] = 5.0
        got = ev.s1_depth(raw)
        assert got.dtype == torch.bfloat16 and got.shape == (224, 224)
        assert torch.equal(got.view(torch.int16), ref.to(torch.bfloat16).view(torch.int16))


def test_s1_rgb_bf16_rounding_is_torch_division():
    """float32 u / 255 rounded to bf16 (the device frame path) == torch's bf16(u8) / 255 for all 256 bytes."""
    u = torch.arange(256, dtype=torch.uint8)
    assert torch.equal((u.float() / 255).to(torch.bfloat16).view(torch.int16), (u.to(torch.bfloat16) / 255).view(torch.int16))


def test_summarize_equals_reference_calc_metrics():
    from internnav_b200.habitat_eval import summarize
    case = GOLDEN["calc_metrics"]
    x = case["inputs"]
    results = [{"success": s, "spl": p, "os": o, "ne": n, "ndtw": d}
               for s, p, o, n, d in zip(x["sucs"], x["spls"], x["oss"], x["nes"], x["ndtws"])]
    got = summarize(results)
    assert got == case["outputs"], (got, case["outputs"])
    assert any(math.isnan(p) for p in x["spls"]) and any(math.isinf(n) for n in x["nes"])
    no_ndtw = summarize([{k: v for k, v in r.items() if k != "ndtw"} for r in results])
    assert "ndtws_all" not in no_ndtw and no_ndtw["sucs_all"] == got["sucs_all"]


def test_conjunctions_match_reference_and_policy_default_is_unchanged():
    from internnav_b200 import policy as P
    from internnav_b200.habitat_eval import CONJUNCTIONS
    assert CONJUNCTIONS == GOLDEN["constants"]["conjunctions"] and P.PROMPT == GOLDEN["constants"]["prompt"]
    assert P.CONJUNCTION == "you can see "
    log = []
    pol = P.InternVLAN1Policy(H.BatchedModel({0: ["↑"]}, {0: log}), H.Processor({0: log}), num_envs=1)
    obs = H.observation(1, 0, 0)
    pol.s2_step([0], [obs["rgb"]], [None], [None], [H.instruction(0, 0)[:-1]], None, [False])
    assert "you can see<image>" in log[0]["s2"]
    pol.reset()
    pol.s2_step([0], [obs["rgb"]], [None], [None], [H.instruction(0, 0)[:-1]], None, [False],
                conjunctions=["ahead of you is "])
    assert "ahead of you is<image>" in log[-1]["s2"] and "you can see" not in log[-1]["s2"]


def test_model_without_system1_is_refused():
    from internnav_b200.habitat_eval import HabitatVLNEvaluator
    model = H.BatchedModel({}, {})
    model.has_system1 = False
    with pytest.raises(ValueError, match="System 1"):
        HabitatVLNEvaluator(model, H.Processor({}), depth_filter=H.depth_filter)
