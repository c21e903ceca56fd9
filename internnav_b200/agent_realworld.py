"""Batched real-world agent: the DualVLN robot loop (`system1 = "nextdit_async"`) for B robots at once.

Mirrors `InternVLAN1AsyncAgent` (internnav/agent/internvla_n1_agent_realworld.py), which the reference's inference demo
and its robot server (scripts/realworld/http_internvla_server.py `eval_dual`) drive one robot at a time.  Per robot the
state machine is the reference's:

  * System 2 runs when `episode_idx - last_s2_idx > plan_step_gap`, on a look-down frame, or when the robot holds
    neither an action answer nor a latent plan (`step` L127-140); otherwise the frame only enters the history
    (`step_no_infer`).  The frame of a System-2 call becomes the pixel-goal frame.
  * An action answer (possibly []) is returned once and dropped; a pixel answer gives `output_pixel` [x, y] and a latent
    plan, which drives System 1 on every following step until the next System-2 call (L141-162).
  * System 1 sees [pixel-goal frame, current frame], each resized to 224 x 224 (Pillow's bicubic) and divided by 255,
    and its trajectories become the float64 [T + 1, 2] mean waypoint path (`traj_to_actions(...,
    use_discrate_action=False)`), not action ids.
  * `serve` is `eval_dual` without Flask: reset if asked, step, and for an answer of exactly [5] step again on the same
    image with look_down set; the result is {"discrete_action": [...]} or {"trajectory": [...], "pixel_goal": [x, y]}.

System 2 -- prompts, image history, look-down turns, the device image path, the K/V pool and the feature pool -- is
`InternVLAN1Policy`.  A step makes one System-2 call for every robot that is due, `serve` at most one more for the robots
that answered [5], and then one `generate_traj` call covers every robot that holds a latent plan.

The System-1 frames, the pixel-goal frames and the `generate_traj` call are `preprocess.System1Inputs`: on a CUDA device
the current frames of all robots that need System 1 are resized in one `FramePreprocessor` call, on the CPU with Pillow,
as in the reference.  Depth is resized (no scaling, no clip) only for a System 1 that reads it (`navdp_async`);
`nextdit_async` does not.  The reference hands System 1 float64 frames; this library's System 1 takes float32, which
holds x / 255 of every byte exactly as the reference's `generate_traj` consumes it after its own conversion.

Deviations from the reference class:
  * nothing is written to `save_dir` (no debug images, no answer files) and nothing is printed;
  * the K/V cache of a robot's last System-2 conversation is reused on its look-down turn (byte-identical output, see
    InternVLAN1Policy);
  * an error in one robot's answer (e.g. a lone number, which the reference's pixel parsing cannot read) is returned as
    the Exception in that robot's slot, and the other robots carry on; the reference's single-robot server would raise.
    The failed robot's state is what the reference leaves behind when `step` raises.
"""
import numpy as np
import torch

from . import policy as P
from .postprocess import batched_traj_to_waypoints
from .preprocess import FramePreprocessor, System1Inputs

LOOK_DOWN = [5]


class S2Output(P.S2Output):
    """One robot's result of `step` (the reference's vln_utils.S2Output fields the agent sets): `output_action` (list of
    action ids, possibly []), or `output_trajectory` (float64 numpy [T + 1, 2]); `output_pixel` [x, y] on the step whose
    System-2 call answered with a pixel goal."""

    def __init__(self):
        super().__init__()
        self.output_trajectory = None


class _Robot:
    """What System 2 last told one robot (the reference's output_action / output_latent / output_pixel and
    last_s2_idx)."""
    __slots__ = ("last_s2_idx", "action", "latent", "pixel")

    def __init__(self):
        self.last_s2_idx = -100
        self.action = self.latent = self.pixel = None


class InternVLAN1AsyncAgent:
    def __init__(self, args, model=None, processor=None, num_envs=1, x_init=None, vision_cache_frames=0,
                 kv_pool_tokens=None):
        """args: the reference's (`device`, `model_path`, `resize_w`, `resize_h`, `num_history`, `plan_step_gap`; the gap
        may also be a sequence, one per robot).  Without
        `model` / `processor` the checkpoint at args.model_path is loaded, as the reference does.  `x_init`: None (System 1
        draws its initial noise on the device) or a callable env_ids -> noise [len(env_ids) * 32, T, 3] for those robots,
        in that order.  `vision_cache_frames`, `kv_pool_tokens`: see InternVLAN1Policy."""
        self.device = torch.device(args.device)
        if model is None:
            from .internvla_n1 import InternVLAN1ForCausalLM
            model = InternVLAN1ForCausalLM.from_pretrained(args.model_path, torch_dtype=torch.bfloat16,
                                                           attn_implementation="flash_attention_2",
                                                           device_map={"": self.device})
        if processor is None:
            from transformers import AutoProcessor
            processor = AutoProcessor.from_pretrained(args.model_path)
        processor.tokenizer.padding_side = "left"
        if not getattr(model, "has_system1", True):
            raise ValueError("InternVLAN1AsyncAgent needs a model with a System 1 (the DualVLN checkpoint); this one has "
                             "none: serve it with InternVLAN1Policy")
        self.model, self.processor = model, processor
        self.num_envs = int(num_envs)
        self.plan_step_gap = np.broadcast_to(np.asarray(args.plan_step_gap, dtype=np.int64), (self.num_envs,))
        self.policy = P.InternVLAN1Policy(model, processor, num_envs=num_envs, num_history=args.num_history,
                                          resize_w=args.resize_w, resize_h=args.resize_h, device=self.device,
                                          vision_cache_frames=vision_cache_frames, kv_pool_tokens=kv_pool_tokens)
        self.reads_depth = getattr(getattr(model, "config", None), "system1", None) == "navdp_async"
        self._frames = FramePreprocessor(self.device) if self.device.type == "cuda" else None
        self.s1 = System1Inputs(model, self._frames, x_init)
        self.robots = [_Robot() for _ in range(num_envs)]
        self.calls = {"s2": 0, "s1": 0}

    def reset(self, env_ids=None):
        envs = range(self.num_envs) if env_ids is None else [int(e) for e in env_ids]
        for e in envs:
            self.robots[e] = _Robot()
        self.policy.reset(list(envs))
        self.s1.reset(envs)

    # ------------------------------------------------------------------ L127-164
    def step(self, env_ids, rgbs, depths, poses, instructions, intrinsic=None, look_downs=None):
        """One frame for each listed robot (rgb uint8 [H, W, 3], depth float32 [H, W]) -> one S2Output per robot, or the
        Exception its System-2 answer raised."""
        look_downs = [False] * len(env_ids) if look_downs is None else [bool(v) for v in look_downs]
        outs, goals = self._system2(env_ids, rgbs, depths, poses, instructions, intrinsic, look_downs)
        self._system1(env_ids, rgbs, depths, outs, goals)
        return outs

    def serve(self, env_ids, rgbs, depths, instructions, resets=None, intrinsic=None, poses=None):
        """`eval_dual` (http_internvla_server.py L41-74) for each listed robot -> its JSON-shaped result dict
        ({"discrete_action": ids} or {"trajectory": [[x, y], ...], "pixel_goal": [x, y]}), or the Exception its System-2
        answer raised.  `resets[j]` starts robot env_ids[j]'s episode first."""
        n = len(env_ids)
        if resets is not None and any(resets):
            self.reset([e for e, r in zip(env_ids, resets) if r])
        poses = [np.eye(4) for _ in range(n)] if poses is None else poses
        outs, goals = self._system2(env_ids, rgbs, depths, poses, instructions, intrinsic, [False] * n)
        retry = [j for j in range(n) if not isinstance(outs[j], Exception) and self.robots[env_ids[j]].action == LOOK_DOWN]
        if retry:   # the [5] answer is returned (and dropped) by the first step; the look-down step continues the turn
            for j in retry:
                self.robots[env_ids[j]].action = None
            pick = lambda xs: [xs[j] for j in retry]  # noqa: E731
            again, goals2 = self._system2(pick(env_ids), pick(rgbs), pick(depths), pick(poses), pick(instructions),
                                          intrinsic, [True] * len(retry))
            for j, o in zip(retry, again):
                outs[j] = o
            goals |= goals2
        self._system1(env_ids, rgbs, depths, outs, goals)
        return [o if isinstance(o, Exception) else self._json(o) for o in outs]

    @staticmethod
    def _json(out):
        if out.output_action is not None:
            return {"discrete_action": list(out.output_action)}
        res = {"trajectory": out.output_trajectory.tolist()}
        if out.output_pixel is not None:
            res["pixel_goal"] = list(out.output_pixel)
        return res

    # ------------------------------------------------------------------ System 2
    def _system2(self, env_ids, rgbs, depths, poses, instructions, intrinsic, look_downs):
        """The scheduling half of `step`: history frames for the robots that are not due, one System-2 call for those
        that are.  -> (outputs, env ids whose pixel-goal frame is this step's frame)."""
        outs = [S2Output() for _ in env_ids]
        due, rest = [], []
        for j, e in enumerate(env_ids):
            r = self.robots[e]
            gap = self.policy.episodes[e].episode_idx - r.last_s2_idx > self.plan_step_gap[e]
            (due if gap or look_downs[j] or (r.action is None and r.latent is None) else rest).append(j)
        if rest:
            self.policy.step_no_infer([env_ids[j] for j in rest], [rgbs[j] for j in rest])
        goals = set()
        if not due:
            return outs, goals
        pick = lambda xs: [xs[j] for j in due]  # noqa: E731
        res = self.policy.s2_step(pick(env_ids), pick(rgbs), pick(depths), pick(poses), pick(instructions), intrinsic,
                                  pick(look_downs))
        self.calls["s2"] += 1
        for j, r in zip(due, res):
            if isinstance(r, Exception):
                outs[j] = r
                continue
            e = env_ids[j]
            robot = self.robots[e]
            robot.action, robot.latent = r.output_action, r.output_latent
            robot.pixel = None if r.output_pixel is None else [int(v) for v in r.output_pixel]
            robot.last_s2_idx = self.policy.episodes[e].episode_idx
            outs[j].output_pixel = robot.pixel
            goals.add(e)
        return outs, goals

    # ------------------------------------------------------------------ System 1
    def _system1(self, env_ids, rgbs, depths, outs, goals):
        """The output half of `step`: held action answers are returned once; every robot holding a latent plan gets its
        waypoint path from one generate_traj call."""
        s1 = []
        for j, e in enumerate(env_ids):
            if isinstance(outs[j], Exception):
                continue
            r = self.robots[e]
            if r.action is not None:
                outs[j].output_action, r.action = list(r.action), None
            elif r.latent is not None:
                s1.append(j)
        if not s1:
            return
        envs = [env_ids[j] for j in s1]
        cur = self.s1.rgb([rgbs[j] for j in s1])
        cur_d = self.s1.depth([depths[j] for j in s1]) if self.reads_depth else None
        traj = self.s1.generate(envs, goals, cur, cur_d, [self.robots[e].latent for e in envs])
        self.calls["s1"] += 1
        paths = batched_traj_to_waypoints(traj, len(envs))
        for k, j in enumerate(s1):
            outs[j].output_trajectory = paths[k]
