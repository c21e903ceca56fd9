"""Generate tests/golden/habitat_dialog_traces.json from the REFERENCE's own VL-LN dialog loop -- build container only.

    python -m oracle.gen_golden_dialog

internnav/agent/dialog_agent.py and internnav/habitat_extensions/vlln/habitat_dialog_evaluator.py are imported
untouched, with the modules this container lacks stubbed in sys.modules (habitat, habitat_baselines, quaternion,
depth_camera_filtering, transformers, the registries, the measures, SimpleNPC and get_description).  A real
`DialogAgent` is built from a stub config whose `AutoProcessor` / `AutoTokenizer` / `Qwen2_5_VLForConditionalGeneration`
return the scripted processor and model of oracle/habitat_dialog_script.py, its device set to the CPU, and
`HabitatDialogEvaluator.eval_action` is called unbound on a stand-in `self` holding that agent, the scripted environment
and NPC, in a temporary directory (the loop writes check_sim images, action logs, scene summaries it reads and
progress.json).  The module globals ShortestPathFollower, quaternion (numpy-quaternion's `as_rotation_matrix`),
filter_depth and get_description are the scripted ones; `random` is seeded per case.

Cases: `instance_dialog` with `dialog_enabled`, no `append_look_down`, 5 questions per episode; `objectnav` with
`append_look_down` and no dialog; one `coin` case.  Recorded per case, in order: every environment reset and step (the
agent's own LOOKUP steps included), every System-2 call (chat text, image digests, continued-conversation flag), every
navmesh query, every follower call (goal as exact float64 reprs), every NPC question and answer, then the episode dicts.
A look-down turn whose conversation an action step has cleared ends the reference's run (the processor refuses the
placeholders); that episode's dict is built from the loop's locals at the raise.  Also recorded: the camera-to-episodic
transform and lifted point of every pixel answer, and `calc_metrics` on a set of results with NaN SPL and infinite
errors.
"""
import contextlib
import importlib
import io
import json
import os
import random
import sys
import tempfile
import types
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import habitat_dialog_script as D  # noqa: E402
from oracle import habitat_s2_script as S  # noqa: E402
from oracle import habitat_script as H  # noqa: E402
from oracle import realworld_script as R  # noqa: E402
from oracle.gen_golden_habitat import _module  # noqa: E402
from oracle.ref_loader import REF, available  # noqa: E402

CASES = [
    dict(robot=0, seed=71, episodes=3, task="instance_dialog", dialog_enabled=True, append_look_down=False, turn=5,
         talk=0.3),
    dict(robot=1, seed=72, episodes=3, task="instance_dialog", dialog_enabled=True, append_look_down=False, turn=5,
         talk=0.45, p_number=0.04),
    dict(robot=2, seed=73, episodes=3, task="instance_dialog", dialog_enabled=True, append_look_down=False, turn=5,
         talk=0.2, p_outside=0.06),
    dict(robot=3, seed=74, episodes=4, task="objectnav", dialog_enabled=False, append_look_down=True, turn=5,
         talk=0.0, p_number=0.03),
    dict(robot=4, seed=75, episodes=4, task="objectnav", dialog_enabled=False, append_look_down=True, turn=5,
         talk=0.0, p_outside=0.05, p_reset_down=0.08),
    dict(robot=5, seed=76, episodes=3, task="coin", dialog_enabled=False, append_look_down=False, turn=5, talk=0.0),
]
STUBBED = ("internnav", "habitat", "habitat_baselines", "quaternion", "depth_camera_filtering", "transformers")


def load_reference():
    """(dialog_agent, habitat_dialog_evaluator) modules of the reference, untouched, with their imports stubbed."""
    if not available():
        raise RuntimeError("reference tree not present at %s" % REF)
    saved = {k: sys.modules.get(k) for k in list(sys.modules) if k.split(".")[0] in STUBBED}
    for k in saved:
        del sys.modules[k]
    try:
        for name, rel in [("internnav", ""), ("internnav.agent", "agent"), ("internnav.configs", "configs"),
                          ("internnav.habitat_extensions", "habitat_extensions"),
                          ("internnav.habitat_extensions.vlln", "habitat_extensions/vlln"),
                          ("internnav.habitat_extensions.vlln.simple_npc", "habitat_extensions/vlln/simple_npc"),
                          ("internnav.habitat_extensions.vlln.utils", "habitat_extensions/vlln/utils")]:
            _module(name, os.path.join(REF, "internnav", rel))
        sys.modules["internnav.agent"].Agent = type("Agent", (), {"register": staticmethod(lambda name: (lambda c: c))})
        _module("internnav.configs.agent", AgentCfg=object)
        _module("internnav.configs.evaluator", EvalCfg=object)
        _module("internnav.evaluator", DistributedEvaluator=object,
                Evaluator=SimpleNamespace(register=lambda name: (lambda cls: cls)))
        _module("internnav.habitat_extensions.vlln.measures")
        _module("internnav.habitat_extensions.vlln.simple_npc.simple_npc", SimpleNPC=None)
        _module("internnav.habitat_extensions.vlln.utils.dialog_utils", get_description=None)
        _module("habitat", path="", config=None)
        _module("habitat.config", path="", read_write=contextlib.nullcontext)
        _module("habitat.config.default_structured_configs", CollisionsMeasurementConfig=object, FogOfWarConfig=object,
                TopDownMapMeasurementConfig=object)
        for name in ("habitat.tasks", "habitat.tasks.nav", "habitat.utils", "habitat.utils.visualizations"):
            _module(name, path="")
        _module("habitat.tasks.nav.shortest_path_follower", ShortestPathFollower=None)
        _module("habitat.utils.visualizations.utils", images_to_video=None, observations_to_image=None)
        _module("habitat_baselines", path="")
        _module("habitat_baselines.config", path="")
        _module("habitat_baselines.config.default", get_config=None)
        _module("quaternion")
        _module("depth_camera_filtering", filter_depth=None)
        _module("transformers", AutoProcessor=None, AutoTokenizer=None, Qwen2_5_VLForConditionalGeneration=None)
        with contextlib.redirect_stdout(io.StringIO()):
            agent = importlib.import_module("internnav.agent.dialog_agent")
            evaluator = importlib.import_module("internnav.habitat_extensions.vlln.habitat_dialog_evaluator")
        return agent, evaluator
    finally:
        for k in [k for k in sys.modules if k.split(".")[0] in STUBBED]:
            del sys.modules[k]
        sys.modules.update({k: v for k, v in saved.items() if v is not None})


class _NPC:
    """SimpleNPC stand-in: the scripted oracle, logging every question."""

    def __init__(self, log, robot):
        self.log, self.robot, self.k = log, robot, -1

    def answer_question(self, question, instance_id, object_dict, task_done, path_description, mode):
        self.k += 1
        a = D.npc_answer(self.robot, self.k)
        self.log.append({"npc": question, "answer": a})
        return a


def make_agent(agent_mod, case, processor, model):
    sensors = SimpleNamespace(rgb_sensor=SimpleNamespace(position=[0.0, S.CAMERA_HEIGHT, 0.0], width=S.WIDTH,
                                                         height=S.HEIGHT, hfov=S.HFOV),
                              depth_sensor=SimpleNamespace(min_depth=H.MIN_DEPTH, max_depth=H.MAX_DEPTH, width=S.WIDTH,
                                                           hfov=S.HFOV))
    settings = dict(task_name=case["task"], task=case["task"], sim_sensors_config=sensors, model_path="scripted",
                    mode="system2", append_look_down=case["append_look_down"], resize_h=H.RESIZE, resize_w=H.RESIZE,
                    local_rank=0, dialog_enabled=case["dialog_enabled"], num_history=H.NUM_HISTORY, max_new_tokens=128)
    agent_mod.AutoTokenizer = SimpleNamespace(from_pretrained=lambda *a, **k: processor.tokenizer)
    agent_mod.AutoProcessor = SimpleNamespace(from_pretrained=lambda *a, **k: processor)
    agent_mod.Qwen2_5_VLForConditionalGeneration = SimpleNamespace(from_pretrained=lambda *a, **k: model)
    agent = agent_mod.DialogAgent(SimpleNamespace(model_settings=settings, model_name="dialog"))
    agent.device = torch.device("cpu")
    return agent


def instrument(agent_mod, ev_mod, geometry):
    agent_mod.ShortestPathFollower = D.Follower
    agent_mod.quaternion = types.SimpleNamespace(as_rotation_matrix=S.as_rotation_matrix)
    agent_mod.filter_depth = H.depth_filter
    ev_mod.get_description = lambda env, object_dict, region_dict: ("go ahead", 5.0)
    ref_p2g = agent_mod.DialogAgent.pixel_to_gps

    def pixel_to_gps(self, pixel, depth, intrinsic, tf_camera_to_episodic):
        g = {"pixel": [int(v) for v in pixel], "tf": S.reprs(tf_camera_to_episodic)}
        geometry.append(g)
        v, u = pixel
        inside = 0 <= v < depth.shape[0] and 0 <= u < depth.shape[1]
        g["z"] = {"v": repr(float(depth[v, u])), "dtype": str(depth.dtype)} if inside else None
        out = ref_p2g(self, pixel, depth, intrinsic, tf_camera_to_episodic)
        g["out"] = [repr(float(x)) for x in out]
        return out
    agent_mod.DialogAgent.pixel_to_gps = pixel_to_gps
    return ref_p2g


def run_case(agent_mod, ev_mod, case, reuse_buffer=False):
    r = case["robot"]
    ans = D.answers(np.random.Generator(np.random.PCG64(case["seed"])), talk=case["talk"],
                    p_number=case.get("p_number", 0.0), p_outside=case.get("p_outside", 0.0),
                    p_reset_down=case.get("p_reset_down", 0.0))
    logs = {r: []}
    geometry = []
    env = D.DialogEnv(r, case["seed"], case["episodes"], logs[r], task=case["task"], reuse_buffer=reuse_buffer)
    processor = D.Processor(logs)
    ref_p2g = instrument(agent_mod, ev_mod, geometry)
    try:
        agent = make_agent(agent_mod, case, processor, D.ReferenceModel({r: ans}))
        with tempfile.TemporaryDirectory() as tmp:
            for scene in range(len(CASES)):
                os.makedirs(os.path.join(tmp, "summary", "scene%d" % scene))
                for f in ("object_dict.json", "region_dict.json"):
                    with open(os.path.join(tmp, "summary", "scene%d" % scene, f), "w") as fh:
                        fh.write("{}")
            s = SimpleNamespace(max_steps_per_episode=D.MAX_STEPS_PER_EPISODE, scene_summary=os.path.join(tmp, "summary"),
                                output_path=os.path.join(tmp, "out"), task=case["task"], turn=case["turn"],
                                dialog_enabled=case["dialog_enabled"], save_video=False, epoch=0, rank=0, env=env,
                                agent=agent, npc=_NPC(logs[r], r), objectnav_instruction="search for {target_object}.")
            os.makedirs(s.output_path)
            random.seed(case["seed"])
            error = None
            try:
                with contextlib.redirect_stdout(io.StringIO()), contextlib.redirect_stderr(io.StringIO()):
                    ev_mod.HabitatDialogEvaluator.eval_action(s)
            except ValueError as exc:
                tb = exc.__traceback__
                while tb.tb_frame.f_code.co_name != "eval_action":
                    tb = tb.tb_next
                loc, m = tb.tb_frame.f_locals, env.get_metrics()
                error = {"scene_id": loc["scene_id"], "episode_id": loc["episode_id"], "success": m["success"],
                         "spl": m["spl"], "os": m["oracle_success"], "ne": m["distance_to_goal"], "steps": loc["step_id"],
                         "episode_instruction": loc["episode_instruction"], "path": loc["path_list"],
                         "action": loc["action_list"], "object_category": loc["episode"].object_category,
                         "error": type(exc).__name__, "error_message": str(exc)}
            path = os.path.join(s.output_path, "progress.json")
            results = [json.loads(line) for line in open(path)] if os.path.exists(path) else []
    finally:
        agent_mod.DialogAgent.pixel_to_gps = ref_p2g
    if error is not None:
        results.append(error)
    return {"case": case, "answers": ans, "episodes_run": env._i, "events": logs[r], "results": results,
            "geometry": geometry}


def calc_metrics_case(ev_mod):
    rng = np.random.Generator(np.random.PCG64(9))
    n = 19
    res = {"sucs": rng.integers(0, 2, n).astype(float).tolist(), "spls": rng.uniform(0, 1, n).tolist(),
           "oss": rng.integers(0, 2, n).astype(float).tolist(), "nes": rng.uniform(0, 9, n).tolist()}
    res["spls"][2] = res["spls"][7] = float("nan")
    res["nes"][4] = res["nes"][12] = float("inf")
    out = ev_mod.HabitatDialogEvaluator.calc_metrics(None, {k: torch.tensor(v) for k, v in res.items()})
    return {"inputs": res, "outputs": out}


def main(out=None):
    agent_mod, ev_mod = load_reference()
    intrinsic = agent_mod.DialogAgent.get_intrinsic_matrix(None, SimpleNamespace(width=S.WIDTH, height=S.HEIGHT,
                                                                                 hfov=S.HFOV))
    traces = []
    for case in CASES:
        # fresh observation arrays, as habitat returns them: the reference keeps the `obs` of the last evaluator step
        # across its own LOOKUP steps, so with a simulator that renders into one buffer its next call (after an action
        # 7) would see the LOOKUP view; the batched loop copies every observation when it arrives
        t = run_case(agent_mod, ev_mod, case)
        traces.append(t)
        ev = t["events"]
        print("case", case["robot"], case["task"], "events", len(ev), "s2", sum("s2" in e for e in ev),
              "npc", sum("npc" in e for e in ev), "follow", sum("follow" in e for e in ev),
              "episodes", [(x["steps"], x.get("error")) for x in t["results"]])
    out = out or os.path.join(ROOT, "tests", "golden", "habitat_dialog_traces.json")
    with open(out, "w") as fh:
        json.dump({"constants": {"camera_height": S.CAMERA_HEIGHT, "width": S.WIDTH, "height": S.HEIGHT,
                                 "hfov": S.HFOV, "intrinsic": S.reprs(intrinsic)},
                   "traces": traces, "calc_metrics": calc_metrics_case(ev_mod)}, fh, ensure_ascii=False)
    print("wrote", out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main()
