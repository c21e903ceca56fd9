"""Generate tests/golden/habitat_eval_traces.json from the REFERENCE's own VLN-CE dual-system loop -- build container only.

    python -m oracle.gen_golden_habitat

internnav/habitat_extensions/vln/habitat_vln_evaluator.py is imported untouched, with the modules this container lacks
stubbed in sys.modules (habitat, habitat_baselines, imageio, quaternion, depth_camera_filtering, the measures
registration, the evaluator registry and the model module).  `HabitatVLNEvaluator._run_eval_dual_system` is called
unbound on a stand-in `self` carrying a scripted environment, processor and model (oracle/habitat_script.py), the
prompt, conjunctions and action table read from the reference's `__init__` source, and the dual-system config's values
(8 history frames, 384 x 384, depth 0-10 m) with a small step budget.  The loop writes check_sim images and
progress.json, so each case runs in a temporary directory; `random` is seeded per case.

Recorded per case, in order: every environment reset and step, every System-2 call (chat text, image digests,
look-down flag), every System-1 call (latent tag, digests of the bf16 RGB and depth stacks), and the per-episode dicts
(progress.json).  The reference's run ends at an answer it cannot parse; that episode's dict is built from the loop's
locals at the raise, `get_metrics()` and the exception's name and message.  Each case is run twice, with fresh
observation arrays and with an environment that renders every observation into one buffer; the two traces must be
equal.  Also recorded: `calc_metrics` on a set of episode
results with NaN SPL, infinite errors and nDTW.
"""
import ast
import contextlib
import importlib
import io
import json
import os
import random
import sys
import tempfile
import types
from collections import OrderedDict
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import habitat_script as H  # noqa: E402
from oracle.ref_loader import REF, available  # noqa: E402

CASES = [
    dict(robot=0, seed=31, episodes=3, ndtw=True),
    dict(robot=1, seed=32, episodes=3, ndtw=False),
    dict(robot=2, seed=33, episodes=4, ndtw=True),
    dict(robot=3, seed=36, episodes=3, ndtw=True, p_error=0.06),
]
MODULE = "internnav.habitat_extensions.vln.habitat_vln_evaluator"


def _module(name, path=None, **attrs):
    m = types.ModuleType(name)
    if path is not None:
        m.__path__ = [path]
    m.__dict__.update(attrs)
    sys.modules[name] = m
    return m


def load_reference_evaluator():
    """The reference module habitat_vln_evaluator (untouched) with the simulator-side imports stubbed."""
    if not available():
        raise RuntimeError("reference tree not present at %s" % REF)
    saved = {k: sys.modules.get(k) for k in list(sys.modules)
             if k.split(".")[0] in ("internnav", "habitat", "habitat_baselines", "imageio", "quaternion",
                                    "depth_camera_filtering")}
    for k in saved:
        del sys.modules[k]
    try:
        for name, rel in [("internnav", ""), ("internnav.habitat_extensions", "habitat_extensions"),
                          ("internnav.habitat_extensions.vln", "habitat_extensions/vln"), ("internnav.model", "model"),
                          ("internnav.model.basemodel", "model/basemodel"),
                          ("internnav.model.basemodel.internvla_n1", "model/basemodel/internvla_n1"),
                          ("internnav.model.utils", "model/utils"), ("internnav.configs", "configs")]:
            _module(name, os.path.join(REF, "internnav", rel))
        _module("internnav.model.basemodel.internvla_n1.internvla_n1",
                InternVLAN1ForCausalLM=type("InternVLAN1ForCausalLM", (), {}))
        _module("internnav.configs.evaluator", EvalCfg=object)
        _module("internnav.evaluator", DistributedEvaluator=object,
                Evaluator=SimpleNamespace(register=lambda name: (lambda cls: cls)))
        _module("internnav.habitat_extensions.vln.measures")
        _module("habitat", path="", config=None)
        sys.modules["habitat"].config = _module("habitat.config", path="", read_write=contextlib.nullcontext)
        _module("habitat.config.default", get_agent_config=None)
        _module("habitat.config.default_structured_configs", CollisionsMeasurementConfig=object, FogOfWarConfig=object,
                TopDownMapMeasurementConfig=object)
        for name in ("habitat.tasks", "habitat.tasks.nav", "habitat.utils", "habitat.utils.visualizations"):
            _module(name, path="")
        _module("habitat.tasks.nav.shortest_path_follower", ShortestPathFollower=object)
        _module("habitat.utils.visualizations.utils", images_to_video=None, observations_to_image=None)
        _module("habitat_baselines", path="")
        _module("habitat_baselines.config", path="")
        _module("habitat_baselines.config.default", get_config=None)
        _module("imageio")
        _module("quaternion")
        _module("depth_camera_filtering", filter_depth=H.depth_filter)
        return importlib.import_module(MODULE)
    finally:
        for k in [k for k in sys.modules if k.split(".")[0] in ("internnav", "habitat", "habitat_baselines", "imageio",
                                                                "quaternion", "depth_camera_filtering")]:
            del sys.modules[k]
        sys.modules.update({k: v for k, v in saved.items() if v is not None})


def constructor_constants(path):
    """The prompt, conjunctions and action table that HabitatVLNEvaluator.__init__ sets, read from its source."""
    tree = ast.parse(open(path, encoding="utf-8").read())
    init = next(n for c in tree.body if isinstance(c, ast.ClassDef) and c.name == "HabitatVLNEvaluator"
                for n in c.body if isinstance(n, ast.FunctionDef) and n.name == "__init__")
    out = {}
    for node in ast.walk(init):
        if isinstance(node, ast.Assign) and len(node.targets) == 1:
            t = node.targets[0]
            name = t.id if isinstance(t, ast.Name) else (t.attr if isinstance(t, ast.Attribute) else None)
            if name in ("prompt", "conjunctions"):
                out[name] = ast.literal_eval(node.value)
            elif name == "actions2idx":
                out[name] = OrderedDict(ast.literal_eval(node.value.args[0]))
    return out


def stand_in(cls, consts, env, model, processor, out_dir):
    s = SimpleNamespace(
        model=model, processor=processor, env=env, epoch=0, rank=0, output_path=out_dir, save_video=False,
        vis_debug=False, vis_debug_path=out_dir, max_steps_per_episode=H.MAX_STEPS_PER_EPISODE, device="cpu",
        model_args=SimpleNamespace(resize_w=H.RESIZE, resize_h=H.RESIZE, num_history=H.NUM_HISTORY),
        num_history=H.NUM_HISTORY, _min_depth=H.MIN_DEPTH, _max_depth=H.MAX_DEPTH,
        conversation=[{"from": "human", "value": consts["prompt"]}, {"from": "gpt", "value": ""}],
        conjunctions=consts["conjunctions"], actions2idx=consts["actions2idx"])
    s.parse_actions = lambda output: cls.parse_actions(s, output)
    s.resume_from_output_path = lambda: cls.resume_from_output_path(s)
    return s


def run_case(mod, consts, case, reuse_buffer=False):
    r = case["robot"]
    answers = H.answers(np.random.Generator(np.random.PCG64(case["seed"])), p_error=case.get("p_error", 0.0))
    logs = {r: []}
    env = H.ScriptedEnv(r, case["seed"], case["episodes"], logs[r], ndtw=case["ndtw"], reuse_buffer=reuse_buffer)
    model = H.ReferenceModel({r: answers}, logs)
    with tempfile.TemporaryDirectory() as tmp:
        ev = stand_in(mod.HabitatVLNEvaluator, consts, env, model, H.Processor(logs), tmp)
        random.seed(case["seed"])
        error = None
        try:
            with contextlib.redirect_stdout(io.StringIO()), contextlib.redirect_stderr(io.StringIO()):
                mod.HabitatVLNEvaluator._run_eval_dual_system(ev)
        except IndexError as exc:
            tb = exc.__traceback__
            while tb.tb_frame.f_code.co_name != "_run_eval_dual_system":
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
    return {"case": case, "answers": answers, "episodes_run": env._i, "events": logs[r], "results": results}


def calc_metrics_case(mod):
    rng = np.random.Generator(np.random.PCG64(7))
    n = 23
    res = {"sucs": rng.integers(0, 2, n).astype(float).tolist(), "spls": rng.uniform(0, 1, n).tolist(),
           "oss": rng.integers(0, 2, n).astype(float).tolist(), "nes": rng.uniform(0, 9, n).tolist(),
           "ndtws": rng.uniform(0, 1, n).tolist()}
    res["spls"][3] = res["spls"][11] = float("nan")
    res["nes"][5] = float("inf")
    out = mod.HabitatVLNEvaluator.calc_metrics(None, {k: torch.tensor(v) for k, v in res.items()})
    return {"inputs": res, "outputs": out}


def main():
    mod = load_reference_evaluator()
    consts = constructor_constants(os.path.join(REF, *MODULE.split(".")) + ".py")
    traces = []
    for case in CASES:
        t = run_case(mod, consts, case)
        # the reference copies every frame before its next step, so a simulator that renders into one buffer gives it
        # the same trace; the replay tests use both kinds of environment against this one trace
        assert run_case(mod, consts, case, reuse_buffer=True) == t, case
        traces.append(t)
        ev = t["events"]
        print("case", case, "events", len(ev), "s2", sum("s2" in e for e in ev), "s1", sum("s1" in e for e in ev),
              "episodes", [(x["steps"], x.get("error")) for x in t["results"]])
    out = os.path.join(ROOT, "tests", "golden", "habitat_eval_traces.json")
    with open(out, "w") as fh:
        json.dump({"constants": {"prompt": consts["prompt"], "conjunctions": consts["conjunctions"]},
                   "traces": traces, "calc_metrics": calc_metrics_case(mod)}, fh, ensure_ascii=False)
    print("wrote", out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main()
