"""Generate tests/golden/realworld_agent_traces.json from the REFERENCE's own InternVLAN1AsyncAgent -- build container only.

    python -m oracle.gen_golden_realworld

The reference class (internnav/agent/internvla_n1_agent_realworld.py) is imported untouched.  Its model module is
replaced by a stub whose `InternVLAN1ForCausalLM.from_pretrained` returns oracle/realworld_script.ScriptedReferenceModel,
and the module's `AutoProcessor.from_pretrained` returns the scripted processor.  The class writes debug images and text
under `test_data/` in the working directory, so the episodes run in a temporary directory.

Each case is one robot driven the way the reference server drives it (scripts/realworld/http_internvla_server.py
`eval_dual` L41-74): reset when asked, `step`, and if the answer is exactly [5] a second `step` on the same image with
look_down=True.  Recorded per served frame: every `step` call's output (action list, waypoint path, pixel goal, or the
exception it raised), every model call it made (chat text and image digests of System 2 with the look-down flag; latent
tag and frame digest of System 1), and the JSON result the server would return.
"""
import contextlib
import importlib
import io
import json
import os
import sys
import tempfile
import types
from types import SimpleNamespace

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import realworld_script as R  # noqa: E402
from oracle.ref_loader import REF, available  # noqa: E402

CASES = [
    dict(robot=0, seed=21, plan_step_gap=4, steps=36, resets=[]),
    dict(robot=1, seed=22, plan_step_gap=1, steps=30, resets=[13]),
    dict(robot=2, seed=23, plan_step_gap=8, steps=40, resets=[11, 26]),
    dict(robot=3, seed=24, plan_step_gap=4, steps=34, resets=[17], p_error=0.12),
]
NUM_HISTORY, RESIZE = 8, 384


def load_reference_realworld_agent():
    """The reference module internnav.agent.internvla_n1_agent_realworld (class untouched) with the model module stubbed."""
    if not available():
        raise RuntimeError("reference tree not present at %s" % REF)
    saved = {k: sys.modules.get(k) for k in list(sys.modules) if k == "internnav" or k.startswith("internnav.")}
    for k in saved:
        del sys.modules[k]
    try:
        for name, rel in [("internnav", ""), ("internnav.agent", "agent"), ("internnav.model", "model"),
                          ("internnav.model.basemodel", "model/basemodel"),
                          ("internnav.model.basemodel.internvla_n1", "model/basemodel/internvla_n1"),
                          ("internnav.model.utils", "model/utils")]:
            m = types.ModuleType(name)
            m.__path__ = [os.path.join(REF, "internnav", rel)]
            sys.modules[name] = m
        stub = types.ModuleType("internnav.model.basemodel.internvla_n1.internvla_n1")
        stub.InternVLAN1ForCausalLM = type("InternVLAN1ForCausalLM", (), {})
        sys.modules[stub.__name__] = stub
        return importlib.import_module("internnav.agent.internvla_n1_agent_realworld")
    finally:
        for k in [k for k in sys.modules if k == "internnav" or k.startswith("internnav.")]:
            del sys.modules[k]
        sys.modules.update({k: v for k, v in saved.items() if v is not None})


def _output(out):
    return {"action": None if out.output_action is None else [int(a) for a in out.output_action],
            "pixel": None if out.output_pixel is None else [int(v) for v in out.output_pixel],
            "trajectory": None if out.output_trajectory is None else np.asarray(out.output_trajectory).tolist()}


def run_case(mod, case):
    rng = np.random.Generator(np.random.PCG64(case["seed"]))
    answers = R.random_answers(rng, p_error=case.get("p_error", 0.0))
    log = []
    model = R.ScriptedReferenceModel({case["robot"]: answers}, log)
    mod.InternVLAN1ForCausalLM.from_pretrained = staticmethod(lambda *a, **k: model)
    mod.AutoProcessor = SimpleNamespace(from_pretrained=lambda *a, **k: R.ScriptedProcessor(log))
    args = SimpleNamespace(device="cpu", model_path="scripted", resize_w=RESIZE, resize_h=RESIZE, num_history=NUM_HISTORY,
                           plan_step_gap=case["plan_step_gap"])
    agent = mod.InternVLAN1AsyncAgent(args)
    ins = R.instruction(case["robot"])
    frames = []
    for k in range(case["steps"]):
        rgb, depth = R.frame(case["seed"], k)
        reset = k == 0 or k in case["resets"]
        if reset:
            agent.reset()
        steps, look_down, out = [], False, None
        while True:
            del log[:]
            try:
                out = agent.step(rgb, depth, np.eye(4), ins, intrinsic=None, look_down=look_down)
                rec = {"look_down": look_down, "output": _output(out)}
            except Exception as exc:  # noqa: BLE001 -- the server would answer this request with an error
                out = exc
                rec = {"look_down": look_down, "error": type(exc).__name__}
            rec["calls"] = [dict(c, look_down=look_down) if "s2" in c else dict(c) for c in log]
            steps.append(rec)
            if look_down or isinstance(out, Exception) or out.output_action != [5]:
                break
            look_down = True
        if isinstance(out, Exception):
            result = {"error": type(out).__name__}
        elif out.output_action is not None:
            result = {"discrete_action": [int(a) for a in out.output_action]}
        else:
            result = {"trajectory": np.asarray(out.output_trajectory).tolist()}
            if out.output_pixel is not None:
                result["pixel_goal"] = [int(v) for v in out.output_pixel]
        frames.append({"k": k, "reset": reset, "steps": steps, "result": result})
    return {"case": dict(case, num_history=NUM_HISTORY, resize=RESIZE), "answers": answers, "frames": frames}


def main():
    mod = load_reference_realworld_agent()
    traces = []
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        os.chdir(tmp)
        try:
            for case in CASES:
                with contextlib.redirect_stdout(io.StringIO()):   # the reference prints every answer
                    traces.append(run_case(mod, case))
                fr = traces[-1]["frames"]
                kinds = [next(iter(f["result"])) for f in fr]
                print("case", case, {k: kinds.count(k) for k in set(kinds)},
                      "look-down retries", sum(len(f["steps"]) == 2 for f in fr),
                      "s1 calls", sum(1 for f in fr for s in f["steps"] for c in s["calls"] if "s1" in c))
        finally:
            os.chdir(cwd)
    out = os.path.join(ROOT, "tests", "golden", "realworld_agent_traces.json")
    with open(out, "w") as fh:
        json.dump({"traces": traces}, fh, ensure_ascii=False)
    print("wrote", out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main()
