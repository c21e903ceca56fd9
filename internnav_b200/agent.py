"""Batched dual-system agent: when to run System 2, when System 1, what to do with queued actions -- for B environments
at once.

The reference agent (`InternVLAN1Agent`, internnav/agent/internvla_n1_agent.py) serves ONE environment: `step` L243-407
decides per frame whether the S2 worker thread (L133-208) must answer first (`should_infer_s2` L210-241), blocks on it
in 0.5 s / 0.2 s sleep polls (L270-274), then either pops a queued discrete action or runs System 1 on the latent plan
with the goal-frame memory.  Here the same per-environment integer state machine is kept as arrays over the
environments, and each `step` does at most ONE batched System-2 call (all environments that need a new plan this frame)
and ONE batched System-1 call (all environments that must turn a latent plan into actions) -- no worker thread, no
polling: the GPU batch is the concurrency.

Policy interface (duck-typed; `PerEnvPolicies` adapts B single-environment policies with the reference's method names):
    reset(env_ids)
    step_no_infer(env_ids, rgbs, depths, poses)
    s2_step(env_ids, rgbs, depths, poses, instructions, intrinsic, look_downs) -> list of results, one per env; a
        result is an object with output_action / output_pixel / output_latent, or an Exception instance for an
        environment whose call failed (the agent then applies the reference's retry rule L165-189 to that one only)
    s1_step_latent(env_ids, rgbs, depths, latents) -> list of objects with `.idx` (action-id list)
"""
import numpy as np
import torch
from PIL import Image

from .preprocess import SYS1_DEPTH_THRESHOLD   # internvla_n1_agent.py L60

LOOK_DOWN = 5
SYS1_FORWARD_STEP = 4        # internvla_n1_agent.py L61


class PerEnvPolicies:
    """B independent single-environment policies (reference method names) behind the batched interface."""

    def __init__(self, policies):
        self.policies = list(policies)

    def eval(self):
        return self

    def reset(self, env_ids):
        for e in env_ids:
            self.policies[e].reset()

    def step_no_infer(self, env_ids, rgbs, depths, poses):
        for e, r, d, p in zip(env_ids, rgbs, depths, poses):
            self.policies[e].step_no_infer(r, d, p)

    def s2_step(self, env_ids, rgbs, depths, poses, instructions, intrinsic, look_downs):
        out = []
        for e, r, d, p, ins, ld in zip(env_ids, rgbs, depths, poses, instructions, look_downs):
            try:
                out.append(self.policies[e].s2_step(r, d, p, ins, intrinsic, ld))
            except Exception as exc:  # noqa: BLE001 -- the agent owns the retry rule
                out.append(exc)
        return out

    def s1_step_latent(self, env_ids, rgbs, depths, latents):
        return [self.policies[e].s1_step_latent(r, d, lat) for e, r, d, lat in zip(env_ids, rgbs, depths, latents)]


def intrinsic_matrix(width, height, hfov):
    """Pinhole intrinsics [4, 4] of a width x height sensor with horizontal field of view `hfov` degrees (square
    pixels, principal point at the centre of the pixel grid): internvla_n1_agent.py L119-131."""
    fx = (width / 2.0) / np.tan(np.deg2rad(hfov / 2.0))
    return np.array([[fx, 0.0, (width - 1.0) / 2.0, 0.0], [0.0, fx, (height - 1.0) / 2.0, 0.0],
                     [0.0, 0.0, 1.0, 0.0], [0.0, 0.0, 0.0, 1.0]])


def s1_frames(goal_rgb, goal_depth, rgb, depth):
    """System-1 input of one environment in partial_async mode (L308-334): [goal frame, current frame], 224x224,
    RGB / 255, depth x 10 (metres) clipped at 5.  -> (float64 [1, 2, 224, 224, 3], float64 [1, 2, 224, 224, 1])"""
    def f_rgb(x):
        return np.array(Image.fromarray(x).resize((224, 224))) / 255.0

    def f_depth(x):
        d = np.array(Image.fromarray(x[:, :, 0]).resize((224, 224))) * 10.0
        return np.minimum(d, SYS1_DEPTH_THRESHOLD)
    rgbs = torch.from_numpy(np.stack([f_rgb(goal_rgb), f_rgb(rgb)]))[None]
    depths = torch.from_numpy(np.stack([f_depth(goal_depth), f_depth(depth)]))[None, ..., None]
    return rgbs, depths


class _Plan:
    """What System 2 last told one environment (the reference's S2Output, vln_utils.py L150-165)."""
    __slots__ = ("idx", "actions", "pixel", "latent", "rgb", "depth")

    def __init__(self):
        self.idx, self.actions, self.pixel, self.latent, self.rgb, self.depth = -1, None, None, None, None, None

    def empty(self):
        return self.actions is None and self.pixel is None and self.latent is None


class InternVLAN1Agent:
    def __init__(self, policy, num_envs=1, infer_mode="sync", sys2_max_forward_step=8, width=640, height=480, hfov=79,
                 preprocessor=None):
        """`preprocessor`: an internnav_b200.preprocess.FramePreprocessor -- the goal / current frames of all
        environments are then resized on the GPU in one batch (bit-identical to the per-frame Pillow calls of
        `s1_frames`, which stay the default because they need no device)."""
        if infer_mode not in ("sync", "partial_async"):
            raise ValueError("Invalid mode: {}".format(infer_mode))
        self.policy = policy
        self.preprocessor = preprocessor
        self.num_envs = num_envs
        self.mode = infer_mode
        self.sys2_max_forward_step = sys2_max_forward_step
        self.camera_intrinsic = intrinsic_matrix(width, height, hfov)
        self.episode_step = np.zeros(num_envs, dtype=np.int64)
        self.episode_idx = np.zeros(num_envs, dtype=np.int64)
        self.look_down = np.zeros(num_envs, dtype=bool)
        self.dual_forward_step = np.zeros(num_envs, dtype=np.int64)
        self.sys1_infer_times = np.zeros(num_envs, dtype=np.int64)
        self.plans = [_Plan() for _ in range(num_envs)]
        self.calls = {"s2": 0, "s1": 0, "s2_envs": 0, "s1_envs": 0}

    # ------------------------------------------------------------------ episode boundaries (L87-117)
    def reset(self, reset_index=None):
        """reset() before the first episode (episode_idx -> -1 everywhere); reset([i, ...]) when those environments
        start their next episode.  `look_down` deliberately survives, as in the reference."""
        envs = list(range(self.num_envs)) if reset_index is None else [int(i) for i in reset_index]
        for e in envs:
            self.episode_idx[e] = -1 if reset_index is None else self.episode_idx[e] + 1
            self.episode_step[e] = 0
            self.dual_forward_step[e] = 0
            self.sys1_infer_times[e] = 0
            self.plans[e] = _Plan()
        self.policy.reset(envs)

    # ------------------------------------------------------------------ L210-241
    def needs_s2(self):
        """Boolean [B]: which environments must consult System 2 on this frame."""
        need = (self.episode_step == 0) | self.look_down
        for e in range(self.num_envs):
            if need[e]:
                continue
            p = self.plans[e]
            if self.mode == "sync":
                need[e] = p.actions is None
            else:
                need[e] = self.dual_forward_step[e] >= self.sys2_max_forward_step or p.empty()
        return need

    def _consult_s2(self, envs, obs, poses):
        pol, K = self.policy, self.camera_intrinsic
        pick = lambda key: [obs[e][key] for e in envs]  # noqa: E731
        lds = [bool(self.look_down[e]) for e in envs]
        res = pol.s2_step(envs, pick("rgb"), pick("depth"), [poses[e] for e in envs], pick("instruction"), K, lds)
        self.calls["s2"] += 1
        self.calls["s2_envs"] += len(envs)
        for e, r in zip(envs, res):
            if isinstance(r, Exception):           # L165-189: reset, retry once without look_down, else STOP
                pol.reset([e])
                r = pol.s2_step([e], [obs[e]["rgb"]], [obs[e]["depth"]], [poses[e]], [obs[e]["instruction"]], K, [False])[0]
                if isinstance(r, Exception):
                    pol.reset([e])
                    p = self.plans[e]
                    p.pixel, p.actions, p.latent = None, [0], None
                    continue
            p = self.plans[e]
            p.pixel, p.actions, p.latent = r.output_pixel, r.output_action, r.output_latent
            p.idx, p.rgb, p.depth = int(self.episode_step[e]), obs[e]["rgb"], obs[e]["depth"]

    # ------------------------------------------------------------------ L243-407
    def step(self, obs):
        B = self.num_envs
        assert len(obs) == B, "one observation dict per environment"
        poses = [np.eye(4, dtype=np.int64) for _ in range(B)]
        need = self.needs_s2()
        ask = [e for e in range(B) if need[e]]
        skip = [e for e in range(B) if not need[e]]
        if skip:  # frames that do not reach System 2 still enter its image history (L264-266)
            self.policy.step_no_infer(skip, [obs[e]["rgb"] for e in skip], [obs[e]["depth"] for e in skip],
                                      [poses[e] for e in skip])
        if ask:
            self.dual_forward_step[ask] = 0
            self._consult_s2(ask, obs, poses)

        actions = [None] * B
        to_s1 = []
        for e in range(B):
            p = self.plans[e]
            if p.actions is not None:                      # queued discrete actions first (L280-299)
                a = p.actions[0]
                p.actions = p.actions[1:] or None
                if a == LOOK_DOWN:
                    self.look_down[e] = True
                    p.actions = p.pixel = p.latent = None
                    a = -1
                    self.sys1_infer_times[e] = 0
                else:
                    self.look_down[e] = False
                    if self.sys1_infer_times[e] > 0:
                        self.dual_forward_step[e] += 1
                actions[e] = a
            else:
                self.look_down[e] = False
                if p.latent is None:
                    raise AssertionError("S2 output should be either action or latent, but got neither! env %d" % e)
                to_s1.append(e)

        if to_s1:
            if self.mode == "sync":                        # L335
                rgbs = [obs[e]["rgb"] for e in to_s1]
                depths = [obs[e]["depth"] * 10000.0 for e in to_s1]
            elif self.preprocessor is not None:
                r, d = self.preprocessor.s1_frames([self.plans[e].rgb for e in to_s1], [self.plans[e].depth for e in to_s1],
                                                   [obs[e]["rgb"] for e in to_s1], [obs[e]["depth"] for e in to_s1])
                rgbs, depths = [r[j:j + 1] for j in range(len(to_s1))], [d[j:j + 1] for j in range(len(to_s1))]
            else:
                pairs = [s1_frames(self.plans[e].rgb, self.plans[e].depth, obs[e]["rgb"], obs[e]["depth"]) for e in to_s1]
                rgbs, depths = [a for a, _ in pairs], [b for _, b in pairs]
            outs = self.policy.s1_step_latent(to_s1, rgbs, depths, [self.plans[e].latent for e in to_s1])
            self.calls["s1"] += 1
            self.calls["s1_envs"] += len(to_s1)
            for e, o in zip(to_s1, outs):
                idx = list(o.idx)
                p = self.plans[e]
                actions[e] = idx[0] if idx else -1
                p.actions = idx[1:] or None
                p.pixel = None
                if self.mode == "sync":
                    p.latent = None
                else:                                      # L352-367
                    if len(idx) < SYS1_FORWARD_STEP and len(idx) + self.dual_forward_step[e] < self.sys2_max_forward_step:
                        self.dual_forward_step[e] = self.sys2_max_forward_step - len(idx)
                    self.sys1_infer_times[e] += 1
                    self.dual_forward_step[e] += 1

        self.episode_step += 1
        return [{"action": [int(a)], "ideal_flag": True} for a in actions]
