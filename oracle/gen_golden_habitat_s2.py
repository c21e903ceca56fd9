"""Generate tests/golden/habitat_eval_s2_traces.json from the REFERENCE's own VLN-CE system2 loop -- build container only.

    python -m oracle.gen_golden_habitat_s2

internnav/habitat_extensions/vln/habitat_vln_evaluator.py is imported untouched with the simulator-side modules
stubbed, as oracle/gen_golden_habitat.py does.  `HabitatVLNEvaluator._run_eval_system2` is called unbound on a stand-in
`self` carrying the scripted environment, follower, processor and model of oracle/habitat_s2_script.py, the prompt,
conjunctions and action table read from the reference's `__init__` source, and the system2 config's values (8 history
frames, 384 x 384, a 640 x 480 RGB sensor with hfov 79, depth 0-10 m, camera height 1.25 m) with a small step budget.
The module's globals ShortestPathFollower, quaternion (numpy-quaternion's `as_rotation_matrix`) and filter_depth are
the scripted ones; pixel_to_gps and xyz_yaw_pitch_to_tf_matrix are the reference's own (utils.py), wrapped to log.

Recorded per case, in order: every environment reset and step, every System-2 call (chat text, image digests,
look-down flag), every depth frame lifted for a pixel answer (digest of the metre frame, pixel), every navmesh query
and every follower call (goal as exact float64 reprs, answer, return type), then the episode dicts.  An error that ends
the reference's run (a lone number, a point outside the depth frame, a look-down turn whose conversation an action step
has cleared) is recorded as the episode dict built from the loop's locals at the raise.  Also recorded per case: the
reference's filter_depth calls, and per pixel answer the geometry (start-pose quaternion and rotation matrix, camera
position and yaw, camera-to-episodic transform, depth value, lifted point).
"""
import contextlib
import io
import json
import os
import random
import sys
import tempfile
import types
from types import SimpleNamespace

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import habitat_s2_script as S  # noqa: E402
from oracle import habitat_script as H  # noqa: E402
from oracle import realworld_script as R  # noqa: E402
from oracle.gen_golden_habitat import MODULE, constructor_constants, load_reference_evaluator  # noqa: E402
from oracle.ref_loader import REF  # noqa: E402

CASES = [
    dict(robot=0, seed=51, episodes=3, ndtw=True),
    dict(robot=1, seed=52, episodes=3, ndtw=False),
    dict(robot=2, seed=53, episodes=3, ndtw=True),
    dict(robot=3, seed=54, episodes=4, ndtw=True, p_number=0.05),
    dict(robot=4, seed=55, episodes=4, ndtw=True, p_outside=0.05),
    dict(robot=5, seed=63, episodes=4, ndtw=False, p_reset_down=0.1),
]


def typed(v):
    return {"v": reprs1(v), "dtype": str(np.asarray(v).dtype)}


def reprs1(v):
    return S.reprs(v) if np.ndim(v) else repr(float(v))


def stand_in(cls, consts, env, model, processor, out_dir):
    sensor = SimpleNamespace(width=S.WIDTH, height=S.HEIGHT, hfov=S.HFOV)
    s = SimpleNamespace(
        model=model, processor=processor, env=env, epoch=0, rank=0, output_path=out_dir, save_video=False,
        vis_debug=False, vis_debug_path=out_dir, max_steps_per_episode=S.MAX_STEPS_PER_EPISODE, device="cpu",
        model_args=SimpleNamespace(resize_w=H.RESIZE, resize_h=H.RESIZE, num_history=H.NUM_HISTORY),
        num_history=H.NUM_HISTORY, _min_depth=H.MIN_DEPTH, _max_depth=H.MAX_DEPTH, _camera_height=S.CAMERA_HEIGHT,
        config=SimpleNamespace(habitat=SimpleNamespace(simulator=SimpleNamespace(agents=SimpleNamespace(
            main_agent=SimpleNamespace(sim_sensors=SimpleNamespace(rgb_sensor=sensor)))))),
        conversation=[{"from": "human", "value": consts["prompt"]}, {"from": "gpt", "value": ""}],
        conjunctions=consts["conjunctions"], actions2idx=consts["actions2idx"])
    s.parse_actions = lambda output: cls.parse_actions(s, output)
    s.resume_from_output_path = lambda: cls.resume_from_output_path(s)
    return s


def instrument(mod, refs, log, geometry, counts):
    """Point the loop's module globals at the scripted / logging pieces for one case; refs: the reference's own
    (pixel_to_gps, xyz_yaw_pitch_to_tf_matrix)."""
    ref_p2g, ref_tf = refs
    last = {}

    def rotation(q):
        m = S.as_rotation_matrix(q)
        last["start"] = {"quat": S.reprs(q.components()), "rot": S.reprs(m)}
        return m

    def tf(xyz, yaw, pitch):
        last["camera"] = {"xyz": typed(xyz), "yaw": typed(yaw), "pitch": repr(float(pitch))}
        return ref_tf(xyz, yaw, pitch)

    def filter_depth(depth, blur_type=None):
        counts["filter"] += 1
        return H.depth_filter(depth, blur_type=blur_type)

    def pixel_to_gps(pixel, depth, intrinsic, tf_camera_to_episodic):
        log.append({"depth": R.digest(depth), "pixel": [int(v) for v in pixel]})
        g = {"pixel": [int(v) for v in pixel], "tf": S.reprs(tf_camera_to_episodic), **last["start"], **last["camera"]}
        geometry.append(g)
        v, u = pixel
        g["z"] = typed(depth[v, u]) if 0 <= v < depth.shape[0] and 0 <= u < depth.shape[1] else None
        out = ref_p2g(pixel, depth, intrinsic, tf_camera_to_episodic)
        g["out"] = [repr(float(x)) for x in out]
        return out

    mod.ShortestPathFollower = S.ScriptedFollower
    mod.quaternion = types.SimpleNamespace(as_rotation_matrix=rotation)
    mod.filter_depth = filter_depth
    mod.xyz_yaw_pitch_to_tf_matrix = tf
    mod.pixel_to_gps = pixel_to_gps


def run_case(mod, refs, consts, case):
    r = case["robot"]
    ans = S.answers(np.random.Generator(np.random.PCG64(case["seed"])), p_number=case.get("p_number", 0.0),
                    p_outside=case.get("p_outside", 0.0), p_reset_down=case.get("p_reset_down", 0.0))
    logs = {r: []}
    geometry, counts = [], {"filter": 0}
    env = S.ScriptedEnvS2(r, case["seed"], case["episodes"], logs[r], ndtw=case["ndtw"])
    model = H.ReferenceModel({r: ans}, logs)
    instrument(mod, refs, logs[r], geometry, counts)
    with tempfile.TemporaryDirectory() as tmp:
        ev = stand_in(mod.HabitatVLNEvaluator, consts, env, model, S.Processor(logs), tmp)
        random.seed(case["seed"])
        error = None
        try:
            with contextlib.redirect_stdout(io.StringIO()), contextlib.redirect_stderr(io.StringIO()):
                mod.HabitatVLNEvaluator._run_eval_system2(ev)
        except (IndexError, ValueError) as exc:
            tb = exc.__traceback__
            while tb.tb_frame.f_code.co_name != "_run_eval_system2":
                tb = tb.tb_next
            loc, m = tb.tb_frame.f_locals, env.get_metrics()
            error = {"scene_id": loc["scene_id"], "episode_id": loc["episode_id"], "success": m["success"],
                     "spl": m["spl"], "os": m["oracle_success"], "ne": m["distance_to_goal"], "steps": loc["step_id"],
                     "episode_instruction": loc["episode_instruction"]}
            if "ndtw" in m:
                error["ndtw"] = m["ndtw"]
            error["error"], error["error_message"] = type(exc).__name__, str(exc)
        path = os.path.join(tmp, "progress.json")
        results = [json.loads(line) for line in open(path)] if os.path.exists(path) else []
    if error is not None:
        results.append(error)
    return {"case": case, "answers": ans, "episodes_run": env._i, "events": logs[r], "results": results,
            "reference_filter_calls": counts["filter"], "geometry": geometry}


def main(out=None):
    mod = load_reference_evaluator()
    refs = (mod.pixel_to_gps, mod.xyz_yaw_pitch_to_tf_matrix)
    consts = constructor_constants(os.path.join(REF, *MODULE.split(".")) + ".py")
    intrinsic = mod.get_intrinsic_matrix(SimpleNamespace(width=S.WIDTH, height=S.HEIGHT, hfov=S.HFOV))
    traces = []
    for case in CASES:
        t = run_case(mod, refs, consts, case)
        traces.append(t)
        ev = t["events"]
        print("case", case, "events", len(ev), "s2", sum("s2" in e for e in ev),
              "follow", sum("follow" in e for e in ev), "lifted", sum("depth" in e for e in ev),
              "episodes", [(x["steps"], x.get("error")) for x in t["results"]])
    out = out or os.path.join(ROOT, "tests", "golden", "habitat_eval_s2_traces.json")
    with open(out, "w") as fh:
        json.dump({"constants": {"camera_height": S.CAMERA_HEIGHT, "width": S.WIDTH, "height": S.HEIGHT,
                                 "hfov": S.HFOV, "intrinsic": S.reprs(intrinsic),
                                 "axis_align": mod.get_axis_align_matrix().tolist()},
                   "traces": traces}, fh, ensure_ascii=False)
    print("wrote", out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main()
