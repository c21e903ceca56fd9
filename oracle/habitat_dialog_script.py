"""Scripted simulator, follower, NPC, processor and models for the VL-LN dialog / ObjectNav evaluation -- TEST
INFRASTRUCTURE.

Drives the reference's `HabitatDialogEvaluator.eval_action` with its `DialogAgent` (oracle/gen_golden_dialog.py) and the
batched `HabitatDialogEvaluator.run` (internnav_b200/habitat_dialog.py, tests/test_dialog_eval_*.py) with the same
scripted pieces, built on oracle/habitat_s2_script.py, and logs per environment, in order, every environment reset and
step, System-2 call, navmesh query, follower call and NPC question:

  DialogEnv       habitat_s2_script.ScriptedEnvS2 plus what the dialog loop reads: `_env.current_episode` (an instance
                  dialog, ObjectNav or CoIN episode whose text names its robot), `_env.episode_over` and a `semantic`
                  observation;
  Follower        habitat_s2_script.ScriptedFollower answering plain ints (the reference writes its action list as JSON);
  npc_answer      the scripted oracle: answer k of robot r, None for some k;
  ReferenceModel  `generate` of Qwen2.5-VL for one environment (the reference agent's call).

Environment r's prompts name "robot <r>:", so the processor and the models route by it (the realworld_script
convention); it answers with answers[r][n] on its n-th System-2 call.
"""
import hashlib
from types import SimpleNamespace

import numpy as np
import torch

from oracle import habitat_s2_script as S
from oracle import habitat_script as H
from oracle import realworld_script as R

MAX_STEPS_PER_EPISODE = 24
CATEGORIES = ["chair", "potted_plant", "tv_monitor", "bed", "toilet", "sofa"]


class _HabitatEnv:
    """The `env._env` surface the dialog loop reads."""

    def __init__(self, env):
        self.env, self.sim = env, S.ScriptedSim(env)

    @property
    def current_episode(self):
        return self.env.get_current_episode()

    @property
    def episode_over(self):
        return bool(self.env.actions) and self.env.actions[-1] == 0


class DialogEnv(S.ScriptedEnvS2):
    def __init__(self, robot, seed, n_episodes, log, task="instance_dialog", reuse_buffer=False):
        super().__init__(robot, seed, n_episodes, log, ndtw=False, reuse_buffer=reuse_buffer)
        self.task = task
        self._env = _HabitatEnv(self)

    def _observe(self):
        obs = super()._observe()
        obs = dict(obs, semantic=np.zeros((1, 4), dtype=np.int32))
        return obs

    def get_current_episode(self):
        category = "robot_%d:_%s" % (self.robot, CATEGORIES[(self.robot + self.ep) % len(CATEGORIES)])
        text = H.instruction(self.robot, self.ep)
        instruction = text if self.task == "coin" else \
            SimpleNamespace(instruction_text=text, instance_id=["%d_%d" % (self.robot, self.ep)])
        return SimpleNamespace(scene_id="data/scene_datasets/hm3d/scene%d/scene%d.glb" % (self.robot, self.robot),
                               episode_id=str(100 * self.robot + self.ep), object_category=category,
                               instruction=instruction)

    def get_metrics(self):
        m = super().get_metrics()
        m.pop("ndtw", None)
        return m


class Follower(S.ScriptedFollower):
    def get_next_action(self, goal):
        from internnav_b200.habitat_eval import follower_action
        return int(follower_action(super().get_next_action(goal)))


def npc_answer(robot, k):
    """The oracle's k-th answer to robot r (None for some k)."""
    h = int(hashlib.sha1(("%d:%d" % (robot, k)).encode()).hexdigest()[:8], 16)
    if h % 4 == 0:
        return None
    return "The target is %s the %s, %d steps away." % (["behind", "left of", "past"][h % 3],
                                                         ["red door", "kitchen", "stairs"][(h // 3) % 3], h % 7 + 1)


def answers(rng, n=60, talk=0.0, p_number=0.0, p_outside=0.0, p_reset_down=0.0):
    """habitat_s2_script.answers plus (talk) questions to the oracle, "<talk>" before or after the question."""
    base = S.answers(rng, n, p_number=p_number, p_outside=p_outside, p_reset_down=p_reset_down)
    out = []
    for a in base:
        u = rng.random()
        if u < talk:
            q = "Is the target in room %d?" % int(rng.integers(1, 9))
            out.append("<talk>" + q if u < talk / 2 else q + "<talk>")
        else:
            out.append(a)
    return out


class Processor(S.Processor):
    """habitat_s2_script.Processor refusing a chat whose image placeholders do not match its images, as Qwen2.5-VL does
    (a look-down or dialog turn whose conversation has been cleared)."""

    def __call__(self, text, images=None, return_tensors="pt"):
        from internnav_b200.habitat_dialog import CLEARED
        n, k = text[0].count("<image>"), len(images or [])
        if n != k:
            raise ValueError(CLEARED % (n, k))
        return super().__call__(text, images, return_tensors)


class ReferenceModel:
    """Qwen2_5_VLForConditionalGeneration.generate for one environment: prompt ids + the scripted answer + eos."""

    def __init__(self, script):
        self.script, self.device = R._Answers(script), torch.device("cpu")

    def eval(self):
        return self

    def generate(self, input_ids=None, max_new_tokens=128, do_sample=False, **inputs):
        _, ans, _ = self.script.next(input_ids[0].tolist())
        return torch.cat([input_ids, torch.tensor([[R.CHAR0 + ord(c) for c in ans] + [R.EOS]])], dim=1)


# ------------------------------------------------------------------------------------------------ replay of the traces
def evaluator(traces, logs, device="cpu", model=None, **kw):
    from internnav_b200.habitat_dialog import HabitatDialogEvaluator
    c = traces[0]["case"]
    if model is None:
        model = S.S2Model({t["case"]["robot"]: t["answers"] for t in traces}, logs)
        model.device = torch.device(device)
    return HabitatDialogEvaluator(model, Processor(logs), task=c["task"], dialog_enabled=c["dialog_enabled"],
                                  turn=c["turn"], append_look_down=c["append_look_down"], num_history=H.NUM_HISTORY,
                                  resize_w=H.RESIZE, resize_h=H.RESIZE, min_depth=H.MIN_DEPTH, max_depth=H.MAX_DEPTH,
                                  max_steps_per_episode=MAX_STEPS_PER_EPISODE, depth_filter=H.depth_filter,
                                  camera_height=S.CAMERA_HEIGHT, width=S.WIDTH, height=S.HEIGHT, hfov=S.HFOV,
                                  seeds=[t["case"]["seed"] for t in traces],
                                  make_follower=lambda env: Follower(env._env.sim, 0.25, False), **kw)


def scripted_npc(logs, robots):
    """The batched loop's npc callable over the scripted oracle; logs each question as the reference run does."""
    count = {}

    def npc(questions):
        out = []
        for e, env, obs, question in questions:
            r = robots[e]
            k = count[r] = count.get(r, -1) + 1
            a = npc_answer(r, k)
            logs[r].append({"npc": question, "answer": a})
            out.append(a)
        return out
    return npc


def replay(traces, device="cpu", reuse_buffer=False, model=None, **kw):
    """Traces of one configuration side by side in one evaluator (environment j = traces[j]); assert each environment's
    event log and episode dicts.  -> the evaluator."""
    logs = {t["case"]["robot"]: [] for t in traces}
    robots = [t["case"]["robot"] for t in traces]
    if model is not None:
        model.logs = logs
    ev = evaluator(traces, logs, device, model=model, npc=scripted_npc(logs, robots), **kw)
    envs = [DialogEnv(t["case"]["robot"], t["case"]["seed"], t["episodes_run"], logs[t["case"]["robot"]],
                      task=t["case"]["task"], reuse_buffer=reuse_buffer) for t in traces]
    results = ev.run(envs)
    for t, res in zip(traces, results):
        got = logs[t["case"]["robot"]]
        for i, (a, b) in enumerate(zip(got, t["events"])):
            assert a == b, (t["case"], i, a, b)
        assert len(got) == len(t["events"]), (t["case"], len(got), len(t["events"]))
        assert res == t["results"], (t["case"], res, t["results"])
    return ev
