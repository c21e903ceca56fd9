"""Scripted simulator, follower, processor and models for the VLN-CE system2 evaluation -- TEST INFRASTRUCTURE.

Drives the reference's `HabitatVLNEvaluator._run_eval_system2` (oracle/gen_golden_habitat_s2.py) and the batched
evaluator's `run_system2` (internnav_b200/habitat_eval.py, tests/test_habitat_eval_s2_*.py) with the same scripted
pieces, built on oracle/habitat_script.py, and logs per environment, in order, every environment step, System-2 call,
depth frame lifted for a pixel answer, navmesh query and follower call:

  ScriptedEnvS2     habitat_script.ScriptedEnv plus the surface the system2 loop reads: observation `gps` / `compass`
                    (float32) and `_env.sim` with `get_agent_state()` (float32 position whose height changes on some
                    moves, a non-trivial rotation quaternion) and a `pathfinder` that rejects and snaps some goals;
  ScriptedFollower  ShortestPathFollower(sim, 0.25, False) stand-in whose answers depend on the goal, the agent's
                    position and its call count -- STOP at once, STOP on the pixel-goal iteration's second call, STOP
                    after a short run, or never (the forward limit) -- returned as a tensor, an array or an int;
  Processor         habitat_script.Processor that refuses a prompt whose image placeholders do not match its images, as
                    Qwen2.5-VL does (the reference's look-down turn after an action step);
  S2Model           `generate` of the n1b200 model mirror for B environments (System-2-only; `has_system1` settable).

`quaternion.as_rotation_matrix` is stubbed with numpy-quaternion's formula (`as_rotation_matrix` below).
"""
import hashlib
import math
from types import SimpleNamespace

import numpy as np
import torch

from oracle import habitat_script as H
from oracle import realworld_script as R

CAMERA_HEIGHT, WIDTH, HEIGHT, HFOV = 1.25, 640, 480, 79
MAX_STEPS_PER_EPISODE = 24


class Quat:
    """The attributes of a numpy-quaternion quaternion."""

    def __init__(self, w, x, y, z):
        self.w, self.x, self.y, self.z = w, x, y, z

    def components(self):
        return [self.w, self.x, self.y, self.z]


def as_rotation_matrix(q):
    """numpy-quaternion's as_rotation_matrix (the general, squared-norm-divided form) for one quaternion."""
    q = np.array(q.components(), dtype=np.float64)
    n = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]
    m = np.empty((3, 3))
    m[0, 0] = 1.0 - 2 * (q[2] * q[2] + q[3] * q[3]) / n
    m[0, 1] = 2 * (q[1] * q[2] - q[3] * q[0]) / n
    m[0, 2] = 2 * (q[1] * q[3] + q[2] * q[0]) / n
    m[1, 0] = 2 * (q[1] * q[2] + q[3] * q[0]) / n
    m[1, 1] = 1.0 - 2 * (q[1] * q[1] + q[3] * q[3]) / n
    m[1, 2] = 2 * (q[2] * q[3] - q[1] * q[0]) / n
    m[2, 0] = 2 * (q[1] * q[3] - q[2] * q[0]) / n
    m[2, 1] = 2 * (q[2] * q[3] + q[1] * q[0]) / n
    m[2, 2] = 1.0 - 2 * (q[1] * q[1] + q[2] * q[2]) / n
    return m


def reprs(a):
    return [repr(float(v)) for v in np.asarray(a).reshape(-1)]


class ScriptedPathfinder:
    def __init__(self, log):
        self.log = log

    def is_navigable(self, p):
        ok = int(abs(float(p[0])) * 1e4 + abs(float(p[2])) * 1e3) % 3 != 0
        self.log.append({"navigable": reprs(p), "answer": ok})
        return ok

    def snap_point(self, p):
        self.log.append({"snap": reprs(p)})
        return np.array([round(float(p[0]) * 4) / 4, float(p[1]) - 0.05, round(float(p[2]) * 4) / 4], dtype=np.float32)


class ScriptedSim:
    def __init__(self, env):
        self.env, self.pathfinder = env, ScriptedPathfinder(env.log)

    def get_agent_state(self):
        x, y, z, heading = self.env.pose()
        a = 0.5 * heading
        w, qx, qy, qz = math.cos(a), 0.03 * (1 + self.env.ep), math.sin(a), -0.02
        n = math.sqrt(w * w + qx * qx + qy * qy + qz * qz)
        return SimpleNamespace(position=np.array([x, y, z], dtype=np.float32), rotation=Quat(w / n, qx / n, qy / n, qz / n))


class ScriptedEnvS2(H.ScriptedEnv):
    """ScriptedEnv with a pose: FORWARD moves 0.25 m along the heading (and climbs 3 cm on odd episodes of even robots),
    LEFT / RIGHT turn 15 degrees."""

    def __init__(self, *args, **kw):
        super().__init__(*args, **kw)
        self._env = SimpleNamespace(sim=ScriptedSim(self))

    def pose(self):
        x, y, z, heading = 0.4 * self.robot, 0.1 * self.robot, -0.3 * self.ep, 0.3 + 0.1 * self.ep
        for a in self.actions:
            if a == 1:
                x, z = x + 0.25 * math.cos(heading), z - 0.25 * math.sin(heading)
                y += 0.03 if (self.ep % 2 and self.robot % 2 == 0) else 0.0
            elif a in (2, 3):
                heading += math.radians(15) * (1 if a == 2 else -1)
        return x, y, z, heading

    def _observe(self):
        moves = sum(a not in (4, 5) for a in self.actions)
        pitch = self.actions.count(5) - self.actions.count(4)
        obs = H.observation(self.seed, self.ep, moves, pitch)
        x, _, z, heading = self.pose()
        obs["gps"] = np.array([-(z + 0.3 * self.ep), x - 0.4 * self.robot], dtype=np.float32)
        obs["compass"] = np.array([heading - 0.3 - 0.1 * self.ep], dtype=np.float32)
        if self._buffer is None:
            return obs
        for k, v in obs.items():
            if k not in self._buffer:
                self._buffer[k] = np.empty_like(v)
            np.copyto(self._buffer[k], v)
        return dict(self._buffer)


class ScriptedFollower:
    """ShortestPathFollower(sim, goal_radius, return_one_hot) stand-in; logs every call to the environment's log."""

    def __init__(self, sim, goal_radius=0.25, return_one_hot=False):
        self.sim, self.log, self.calls, self.per_goal = sim, sim.env.log, 0, {}

    def get_next_action(self, goal):
        self.calls += 1
        key = reprs(goal)
        h = int(hashlib.sha1(repr(key).encode()).hexdigest()[:8], 16)
        n = self.per_goal[tuple(key)] = self.per_goal.get(tuple(key), 0) + 1
        plan = h % 6
        stop = (plan == 0) or (plan == 1 and n == 2) or (plan == 2 and n >= 3 + (h // 6) % 4)
        x = float(self.sim.get_agent_state().position[0])
        a = 0 if stop else [1, 1, 2, 1, 3][(h // 7 + n + int(abs(x) * 100)) % 5]
        kind = ("tensor", "array", "int")[self.calls % 3]
        self.log.append({"follow": key, "dtype": str(np.asarray(goal).dtype), "answer": a, "as": kind})
        if kind == "tensor":
            return torch.tensor([a])
        return np.array([a]) if kind == "array" else a


def answers(rng, n=60, p_number=0.0, p_outside=0.0, p_reset_down=0.0):
    """Pixel answers "u, v" (mostly inside the 640 x 480 frame), look-down alone, after arrows (p_reset_down) and
    followed by arrows, arrow runs, STOP, an answer without actions, and the two pixel answers the reference cannot
    use: a lone number (p_number) and a point outside the frame (p_outside)."""
    out = []
    for _ in range(n):
        u = rng.random()
        if u < p_number:
            out.append("%d" % int(rng.integers(0, 480)))
            continue
        u -= p_number
        if u < p_outside:
            out.append("%d, %d" % (int(rng.integers(0, 640)), int(rng.integers(480, 700))))
            continue
        u -= p_outside
        if u < p_reset_down:
            out.append("".join(rng.choice(["↑", "←", "→"], size=int(rng.integers(1, 3)))) + "↓")
        elif u < 0.34:
            out.append("%d, %d" % (int(rng.integers(0, WIDTH)), int(rng.integers(0, HEIGHT))))
        elif u < 0.52:
            out.append("↓")
        elif u < 0.56:
            out.append("↓" + "".join(rng.choice(["↑", "←", "→"], size=int(rng.integers(1, 3)))))
        elif u < 0.6:
            out.append("STOP")
        elif u < 0.62:
            out.append("I cannot tell where to go.")
        else:
            out.append("".join(rng.choice(["↑", "←", "→"], size=int(rng.integers(1, 4)))))
    return out


class Processor(H.Processor):
    def __call__(self, text, images=None, return_tensors="pt"):
        n, k = text[0].count("<image>"), len(images or [])
        if n != k:
            raise ValueError("a look-down turn after an action step: the cleared conversation has %d image placeholder "
                             "for %d images" % (n, k))
        return super().__call__(text, images, return_tensors)


class S2Model(R.ScriptedBatchedModel):
    """`generate` of the n1b200 model mirror for B environments; `generate_with_latents` is counted and refused in
    replays (the system2 mode must not run the latent pass)."""

    has_system1 = False
    config = SimpleNamespace(system1=None, n_query=4)

    def __init__(self, script, logs):
        self.script, self.logs, self.latent_calls = R._Answers(script), logs, 0
        self.device = torch.device("cpu")

    def generate(self, prompts, pixel_values, image_grid_thw, max_new_tokens=128, return_dict_in_generate=False, **kw):
        gen = []
        for p in prompts:
            _, ans, _ = self.script.next(p)
            gen.append([R.CHAR0 + ord(c) for c in ans] + [R.EOS])
        return SimpleNamespace(generated=gen, latents=None, sequences=None)

    def generate_with_latents(self, *a, **kw):
        self.latent_calls += 1
        raise AssertionError("the system2 mode ran the latent pass")


# ------------------------------------------------------------------------------------------------ replay of the traces
def evaluator(traces, logs, device="cpu", model=None, **kw):
    from internnav_b200.habitat_eval import HabitatVLNEvaluator
    if model is None:
        model = S2Model({t["case"]["robot"]: t["answers"] for t in traces}, logs)
        model.device = torch.device(device)
    return HabitatVLNEvaluator(model, Processor(logs), mode="system2", num_history=H.NUM_HISTORY, resize_w=H.RESIZE,
                               resize_h=H.RESIZE, min_depth=H.MIN_DEPTH, max_depth=H.MAX_DEPTH,
                               max_steps_per_episode=MAX_STEPS_PER_EPISODE, seeds=[t["case"]["seed"] for t in traces],
                               camera_height=CAMERA_HEIGHT, width=WIDTH, height=HEIGHT, hfov=HFOV,
                               make_follower=lambda env: ScriptedFollower(env._env.sim, 0.25, False), **kw)


def replay(traces, device="cpu", reuse_buffer=False, depth_filter=None, model=None):
    """All traces side by side in one system2 evaluator (environment j = traces[j]); assert each environment's event
    log and episode dicts.  The lifted depth frames are logged by wrapping habitat_eval.pixel_to_gps, attributed to the
    environment being resumed.  -> the evaluator."""
    from internnav_b200 import habitat_eval as HE
    logs = {t["case"]["robot"]: [] for t in traces}
    robots = [t["case"]["robot"] for t in traces]
    current = [None]

    class Logged(HE.HabitatVLNEvaluator):
        def _advance(self, req, e, gen, value):
            current[0] = e
            HE.HabitatVLNEvaluator._advance(req, e, gen, value)

    ev = evaluator(traces, logs, device, model=model, depth_filter=depth_filter or H.depth_filter)
    ev.__class__ = Logged
    if model is not None:
        model.logs = logs
    original = HE.pixel_to_gps

    def logged(pixel, depth, intrinsic, tf):
        logs[robots[current[0]]].append({"depth": R.digest(depth), "pixel": [int(v) for v in pixel]})
        return original(pixel, depth, intrinsic, tf)

    envs = [ScriptedEnvS2(t["case"]["robot"], t["case"]["seed"], t["episodes_run"], logs[t["case"]["robot"]],
                          ndtw=t["case"]["ndtw"], reuse_buffer=reuse_buffer) for t in traces]
    HE.pixel_to_gps = logged
    try:
        results = ev.run_system2(envs)
    finally:
        HE.pixel_to_gps = original
    for t, res in zip(traces, results):
        got = logs[t["case"]["robot"]]
        for i, (a, b) in enumerate(zip(got, t["events"])):
            assert a == b, (t["case"], i, a, b)
        assert len(got) == len(t["events"]), (t["case"], len(got), len(t["events"]))
        assert res == t["results"], (t["case"], res, t["results"])
    return ev
