"""Scripted environments, processor and models for the VLN-CE dual-system evaluation -- TEST INFRASTRUCTURE.

Drives the reference's `HabitatVLNEvaluator._run_eval_dual_system` (oracle/gen_golden_habitat.py) and the batched
evaluator of internnav_b200/habitat_eval.py (tests/test_habitat_eval_*.py) with the same scripted simulator, System 2
and System 1, and logs, per environment and in order, every environment step and every model call:

  ScriptedEnv        the reference's HabitatEnv surface; seeded 480 x 640 RGB and [H, W, 1] normalised depth (some
                     values land exactly on, or one float32 step below, an integer after the evaluator's `* 1000`) that
                     depend only on the pose, like a renderer's: the moves made so far and the camera pitch; ends on
                     STOP; metrics derived from the action history.  With `reuse_buffer` every observation is written
                     into the same arrays, as a simulator that renders into one buffer does;
  Processor          realworld_script.ScriptedProcessor whose log entries go to the environment named in the prompt;
  ReferenceModel     `generate` / `generate_latents` / `generate_traj` of the reference model (one environment);
  BatchedModel       `generate_with_latents` / `generate_traj` of the n1b200 model mirror (navdp_async: reads depth).

Environment r's instructions read "robot <r>: ..."; it answers with answers[r][n] on its n-th System-2 call (the
realworld_script convention), and System 1 returns trajectories drawn from the latent tag and the digests of the bf16 RGB
and depth stacks: no motion (first id 0 -> LEFT), a short path (a later 0 -> System 2 again) or a long one.
"""
import hashlib
from types import SimpleNamespace

import numpy as np
import torch

from oracle import realworld_script as R

HEIGHT, WIDTH = 480, 640
NS, T = 4, 8
NUM_HISTORY, RESIZE, MIN_DEPTH, MAX_DEPTH, MAX_STEPS_PER_EPISODE = 8, 384, 0.0, 10.0, 24


def depth_filter(depth, blur_type=None):
    """Stand-in for depth_camera_filtering.filter_depth: fills far readings (> 0.98) with 0, as a hole filler would."""
    out = np.array(depth, dtype=np.float32, copy=True)
    out[out > 0.98] = 0.0
    return out


def observation(seed, episode, moves, pitch=0):
    """The view after `moves` moves of an episode with the camera `pitch` LOOKDOWN steps down: rgb uint8
    [480, 640, 3], depth float32 [480, 640, 1] in [0, 1]."""
    rng = np.random.Generator(np.random.PCG64([seed, episode, moves, pitch + 100]))
    rgb = rng.integers(0, 256, size=(HEIGHT, WIDTH, 3), dtype=np.uint8)
    depth = rng.uniform(0.0, 1.0, size=(HEIGHT, WIDTH)).astype(np.float32)
    n = rng.integers(1, 10000, size=(HEIGHT, WIDTH))
    on = (n / 10000).astype(np.float32)                       # * 10 * 1000 in float32 lands on or near n
    kind = rng.integers(0, 3, size=(HEIGHT, WIDTH))
    depth = np.where(kind == 1, on, depth)
    depth = np.where(kind == 2, np.nextafter(on, np.float32(0)), depth)
    return {"rgb": rgb, "depth": depth[:, :, None], "gps": np.zeros(2, dtype=np.float32)}


def instruction(robot, episode):
    return "robot %d: walk past the sofa, turn left at hall %d and stop by the door." % (robot, episode)


class ScriptedEnv:
    """HabitatEnv surface (reset / step / is_running / get_current_episode / get_metrics) over `n_episodes` scripted
    episodes.  Appends {"reset": i} and {"step": action} to `log`."""

    def __init__(self, robot, seed, n_episodes, log, ndtw=True, reuse_buffer=False):
        self.robot, self.seed, self.n_episodes, self.log, self.ndtw = robot, seed, n_episodes, log, ndtw
        self.episodes = list(range(n_episodes))
        self.is_running, self._i, self.actions = True, 0, []
        self._buffer = {} if reuse_buffer else None

    def _observe(self):
        moves = sum(a not in (4, 5) for a in self.actions)
        pitch = self.actions.count(5) - self.actions.count(4)
        obs = observation(self.seed, self.ep, moves, pitch)
        if self._buffer is None:
            return obs
        for k, v in obs.items():
            if k not in self._buffer:
                self._buffer[k] = np.empty_like(v)
            np.copyto(self._buffer[k], v)
        return dict(self._buffer)

    def reset(self):
        if self._i >= self.n_episodes:
            self.is_running = False
            return None
        self.ep, self._i, self.actions = self._i, self._i + 1, []
        self.log.append({"reset": self.ep})
        return self._observe()

    def step(self, action):
        a = int(action)
        self.actions.append(a)
        self.log.append({"step": a})
        return self._observe(), 0.0, a == 0, self.get_metrics()

    def get_current_episode(self):
        return SimpleNamespace(scene_id="data/scene_datasets/mp3d/scene%d/scene%d.glb" % (self.robot, self.robot),
                               episode_id=str(100 * self.robot + self.ep),
                               instruction=SimpleNamespace(instruction_text=instruction(self.robot, self.ep)))

    def get_metrics(self):
        fwd = self.actions.count(1)
        turns = self.actions.count(2) + self.actions.count(3)
        stopped = bool(self.actions) and self.actions[-1] == 0
        ne = abs(6 - fwd) * 0.25 + 0.1 * turns
        m = {"success": float(stopped and ne < 1.0), "oracle_success": float(fwd >= 4),
             "distance_to_goal": ne if fwd else float("inf"), "top_down_map": None,
             "spl": float(stopped and ne < 1.0) * 1.5 / max(1.5, 0.25 * fwd)}
        if self.ndtw:
            m["ndtw"] = float(np.exp(-ne / 3.0))
        return m

    def close(self):
        pass


def answers(rng, n=60, p_error=0.0):
    """Pixel goals, arrow runs, look-down (single and double), STOP, an answer without actions, and (p_error) a lone
    number, which the reference's pixel parsing cannot read."""
    out = []
    for _ in range(n):
        u = rng.random()
        if u < p_error:
            out.append("%d" % int(rng.integers(0, 480)))
        elif u < p_error + 0.42:
            out.append("%d, %d" % (int(rng.integers(0, HEIGHT)), int(rng.integers(0, WIDTH))))
        elif u < p_error + 0.56:
            out.append("↓")
        elif u < p_error + 0.62:
            out.append("↓↓")
        elif u < p_error + 0.66:
            out.append("STOP")
        elif u < p_error + 0.68:
            out.append("I cannot tell where to go.")
        else:
            out.append("".join(rng.choice(["↑", "←", "→"], size=int(rng.integers(1, 4)))))
    return out


def digest(t):
    """Digest of a bf16 System-1 stack [1, 2, 224, 224, C] (as float32)."""
    return R.digest(torch.as_tensor(t).detach().cpu().float().numpy())


def trajectory(tag, d_rgb, d_depth):
    """Scripted System-1 output of one environment: fp32 [NS, T, 3] deltas from the tag and the frame digests."""
    seed = int(hashlib.sha1(("%d:%s:%s" % (tag, d_rgb, d_depth)).encode()).hexdigest()[:12], 16)
    rng = np.random.Generator(np.random.PCG64(seed))
    u = rng.random()
    scale = 0.0 if u < 0.15 else (0.25 if u < 0.35 else 1.0)
    fwd = rng.uniform(0.6, 1.4, size=(NS, T, 1)) * scale
    lat = rng.normal(0.0, 0.3, size=(NS, T, 1)) * scale
    yaw = rng.normal(0.0, 0.1, size=(NS, T, 1))
    return torch.from_numpy(np.concatenate([fwd, lat, yaw], axis=-1).astype(np.float32))


class Processor(R.ScriptedProcessor):
    """ScriptedProcessor whose entries go to logs[robot]; each also carries the look-down flag (a continued turn)."""

    def __init__(self, logs):
        self.logs, self._buf = logs, []
        super().__init__(self._buf)

    def __call__(self, text, images=None, return_tensors="pt"):
        out = super().__call__(text, images, return_tensors)
        call = self._buf.pop()
        call["look_down"] = "<|assistant|>" in text[0][:-len("\n<|assistant|>")]
        self.logs[int(R._ROBOT_RE.search(text[0]).group(1))].append(call)
        return out


class ReferenceModel(R.ScriptedReferenceModel):
    """The reference model's three calls for one environment, System 1 logging its bf16 RGB and depth stacks."""

    def __init__(self, script, logs):
        self.script, self.logs, self.tag = R._Answers(script), logs, None
        self.device = torch.device("cpu")

    def generate_traj(self, traj_latents, images_dp, depths_dp=None):
        tag = int(traj_latents.reshape(-1)[0])
        dr, dd = digest(images_dp), digest(depths_dp)
        self.logs[tag // 1000].append({"s1": tag, "rgb": dr, "depth": dd})
        return trajectory(tag, dr, dd)


class BatchedModel(R.ScriptedBatchedModel):
    """The n1b200 model mirror's calls for B environments; System 1 reads depth (navdp_async)."""

    config = SimpleNamespace(system1="navdp_async", n_query=1)

    def __init__(self, script, logs):
        self.script, self.logs = R._Answers(script), logs
        self.device = torch.device("cpu")

    def generate_traj(self, traj_latents, images_dp, depths_dp=None, x_init=None):
        assert images_dp.dtype == torch.bfloat16 and depths_dp.dtype == torch.bfloat16
        out = []
        for b in range(traj_latents.shape[0]):
            tag = int(traj_latents[b].reshape(-1)[0])
            dr, dd = digest(images_dp[b:b + 1]), digest(depths_dp[b:b + 1])
            self.logs[tag // 1000].append({"s1": tag, "rgb": dr, "depth": dd})
            out.append(trajectory(tag, dr, dd))
        return torch.cat(out).to(images_dp.device)


# ------------------------------------------------------------------------------------------------ replay of the traces
def replay(traces, device="cpu", reuse_buffer=False):
    """All traces side by side in one evaluator (environment j = traces[j]); assert each environment's event log
    (environment steps and model calls, in order) and its episode dicts.  `reuse_buffer`: the environments render
    into one buffer each.  -> the evaluator."""
    from internnav_b200.habitat_eval import HabitatVLNEvaluator
    logs = {t["case"]["robot"]: [] for t in traces}
    model = BatchedModel({t["case"]["robot"]: t["answers"] for t in traces}, logs)
    model.device = torch.device(device)
    ev = HabitatVLNEvaluator(model, Processor(logs), num_history=NUM_HISTORY, resize_w=RESIZE, resize_h=RESIZE,
                             min_depth=MIN_DEPTH, max_depth=MAX_DEPTH, max_steps_per_episode=MAX_STEPS_PER_EPISODE,
                             depth_filter=depth_filter, seeds=[t["case"]["seed"] for t in traces])
    envs = [ScriptedEnv(t["case"]["robot"], t["case"]["seed"], t["episodes_run"], logs[t["case"]["robot"]],
                        ndtw=t["case"]["ndtw"], reuse_buffer=reuse_buffer) for t in traces]
    results = ev.run_dual_system(envs)
    for t, res in zip(traces, results):
        r = t["case"]["robot"]
        got = logs[r]
        assert len(got) == len(t["events"]), (t["case"], len(got), len(t["events"]))
        for i, (a, b) in enumerate(zip(got, t["events"])):
            assert a == b, (t["case"], i, a, b)
        assert res == t["results"], t["case"]
    return ev
