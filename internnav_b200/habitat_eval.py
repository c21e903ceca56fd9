"""Batched VLN-CE evaluation: the dual-system episode loop of the Habitat evaluator for B environments at once.

Mirrors `HabitatVLNEvaluator._run_eval_dual_system` (internnav/habitat_extensions/vln/habitat_vln_evaluator.py L262-629),
the loop behind the reference's R2R-CE / RxR-CE numbers, which runs one environment per process.  Per environment the
loop is the reference's, transcribed as a generator (`_episodes`) that steps its own environment and yields wherever the
reference calls the model:

  * every step that does not follow a LOOKDOWN takes the look-down view: LOOKDOWN twice, keep that observation, LOOKUP
    twice (L346-368); after a pixel-goal answer the camera steps LOOKUP twice more (L440-441);
  * System 2 is asked when no action answer and no pixel goal is held (L370-482), with a conjunction drawn from the
    environment's own `random.Random` (L398) and the instruction without its last character (L381-383); the
    conversation continues after a LOOKDOWN step and starts over after any other step;
  * System 1 sees [pixel-goal look-down frame, current look-down frame]; its action ids (`traj_to_actions`) are padded
    to MAX_STEPS = 8 and cut to MAX_LOCAL_STEPS = 4, zeros kept, and it runs again when the chunk is used up.  A first
    id 0 steps LEFT and drops the goal; a later 0, or more than 8 forward actions on one goal, drops the goal and asks
    System 2 again on the same observation without an environment step (L443-528);
  * an episode ends on `done` or after `max_steps_per_episode` steps and gives the `progress.json` dict (L590-601).

`run_dual_system` drives B such generators in rounds.  A round advances every environment to its next model request,
adds the frames that entered the histories since the last call in one `step_no_infer`, serves every System-2 request in
ONE `InternVLAN1Policy.s2_step` call, resumes those environments (a pixel answer goes straight on to System 1), and serves
every System-1 request in ONE `generate_traj` call followed by `batched_traj_to_actions(..., max_actions=4)`.  An
environment whose episode ends resets and goes on with its next episode in the same round.

System 2 -- prompts, image history, look-down turns, the device image path, the K/V and feature pools -- is
`InternVLAN1Policy`.  The System-1 RGB frames, the pixel-goal frames and the `generate_traj` call are
`preprocess.System1Inputs`: the RGB frames of a round are resized in one call (`FramePreprocessor` on a CUDA device,
Pillow on the CPU) to float32 u / 255 and cast to bf16, which is torch's `bf16(u8) / 255` for every byte.  Depth is
prepared only for a System 1 that reads it (`navdp_async`), on the host: `depth_filter` runs on the full frame, as in
the reference; then only the 224 x 224 source pixels of Pillow's NEAREST resize are taken (`nearest_index`) and the
affine, `* 1000`, the uint16 truncation, `/ 1000`, float32, the clip at 5 and bf16 are applied to those samples.  Every
step after the filter is element-wise, so this is the reference's full-frame path bit for bit.

Deviations from the reference loop:
  * nothing is written (no check_sim images, videos, progress.json or resume) and nothing is printed; the caller
    writes the returned dicts;
  * a look-down turn continues its conversation on the K/V cache (byte-identical output, see InternVLAN1Policy);
  * the pixel goal's latent plan comes from the generate pass's cache instead of a second prefill (`generate_with_latents`);
  * an answer the reference cannot parse (a lone number: IndexError at L436, which ends the reference's run) ends that
    environment's episode; its dict holds `get_metrics()` at that point, the exception's type name under "error" and its
    message under "error_message" (so every dict stays JSON-serialisable), and the other environments carry on;
  * `depth_filter` is supplied by the caller (the reference calls `depth_camera_filtering.filter_depth`).

`HabitatVLNEvaluator(mode="system2").run_system2(envs)` mirrors the evaluator's other mode, `_run_eval_system2`
(L631-945), the benchmark loop of the System-2-only checkpoint, in the same way (`_episodes_system2`):

  * there is no look-down view on every step: the camera tilts only when System 2 answers "↓" (LOOKDOWN twice, no
    step counted, the conversation kept), and the next call is the look-down turn on the full-size frame; every other
    environment step clears the conversation (L877-885);
  * a pixel answer [c0, c1] is the image point (u, v) = (c0, c1): the camera steps LOOKUP twice, the point is lifted
    with that iteration's depth (filter, affine, `* 1000`, `/ 1000`) through the intrinsics and a camera pose built from
    gps, compass, the camera height plus the agent's height change and a 30 degree pitch (`pixel_to_gps`, L706-719 /
    L804), taken to the world frame by the episode-start agent pose and snapped to the navmesh unless navigable
    (L806-809) -- float64 numpy, the reference's operations in its order;
  * the caller's ShortestPathFollower then walks to that goal: on the pixel-goal iteration `get_next_action` is called
    twice (a STOP on the first steps LEFT, drops the goal and clears the conversation); after that once per step, and
    more than MAX_STEPS calls or a STOP drop the goal and count a step without an environment step, so the next
    iteration shows System 2 the same observation, which enters the history again (L811-848).

`run_system2` serves every waiting environment in ONE `s2_step` per round, on `generate` alone (`system2_only`: no
latent pass, whatever the model carries).  Its deviations are those above, plus two:
  * depth is filtered only when a pixel answer needs it (the reference filters every frame and uses the result only
    there; the filter is a function of the one frame, so the goals are the same);
  * a pixel answer the reference cannot use -- a lone number (IndexError at L797) or a point outside the depth frame
    (IndexError in `pixel_to_gps`) -- and a look-down turn whose conversation an action step of the same answer has
    cleared (e.g. "←↓": the reference sends one image placeholder with all of the conversation's images, which
    Qwen2.5-VL refuses) end that environment's episode with `error` / `error_message`.
"""
import random

import numpy as np
import torch

from . import policy as P
from .agent import intrinsic_matrix
from .postprocess import batched_traj_to_actions
from .preprocess import S1_SIZE, SYS1_DEPTH_THRESHOLD, FramePreprocessor, System1Inputs

MAX_STEPS, MAX_LOCAL_STEPS = 8, 4
STOP, FORWARD, LEFT, RIGHT, LOOKUP, LOOKDOWN = range(6)
CAMERA_PITCH = np.deg2rad(30)      # the pitch the system2 loop assumes for every pixel answer (L718)
FOLLOWER_RADIUS = 0.25             # ShortestPathFollower(sim, 0.25, False), once per episode (L663)
CONJUNCTIONS = ["you can see ", "in front of you is ", "there is ", "you can spot ", "you are toward the ",
                "ahead of you is ", "in your sight is "]


def nearest_index(n_in, n_out):
    """Source index of each output pixel of Pillow's NEAREST resize along one axis: int((x + 0.5) * scale) with the
    scale n_in / n_out computed first, in double (Pillow's affine nearest transform).  Multiplying by n_in before
    dividing rounds differently for some sizes."""
    scale = n_in / n_out
    return np.array([int((x + 0.5) * scale) for x in range(n_out)], dtype=np.int64)


def summarize(results):
    """`calc_metrics` (L202-233) over a list of per-episode result dicts: means of success, SPL (NaN / inf count as 0), oracle
    success, the finite navigation errors, and nDTW over the episodes that carry it.  Means are float32, as the
    reference takes them over torch tensors (an empty list gives NaN)."""
    mean = lambda xs: float(torch.tensor(xs, dtype=torch.float32).mean().item())  # noqa: E731
    spl = [float(r["spl"]) if np.isfinite(r["spl"]) else 0.0 for r in results]
    out = {"sucs_all": mean([float(r["success"]) for r in results]), "spls_all": mean(spl),
           "oss_all": mean([float(r["os"]) for r in results]),
           "nes_all": mean([float(r["ne"]) for r in results if np.isfinite(r["ne"])])}
    ndtw = [float(r["ndtw"]) for r in results if "ndtw" in r]
    if ndtw:
        out["ndtws_all"] = mean(ndtw)
    return out


# ---------------------------------------------------------------------------------------------- system2 geometry
# Float64 numpy in the operations, shapes and order of the reference's internnav/habitat_extensions/vln/utils.py
# (get_intrinsic_matrix, xyz_yaw_pitch_to_tf_matrix, get_axis_align_matrix, pixel_to_gps), so that every goal is the
# reference's bit for bit.
AXIS_ALIGN = np.array([[0, 0, 1, 0], [-1, 0, 0, 0], [0, -1, 0, 0], [0, 0, 0, 1]])


def rotation_matrix(q):
    """numpy-quaternion's `as_rotation_matrix` for one quaternion (w, x, y, z attributes, as habitat's agent rotation
    has, or a scalar-first 4-sequence) -> float64 [3, 3]; a non-unit quaternion is divided by its squared norm."""
    w, x, y, z = (q.w, q.x, q.y, q.z) if hasattr(q, "w") else tuple(q)
    w, x, y, z = float(w), float(x), float(y), float(z)
    n = w * w + x * x + y * y + z * z
    if n == 0.0:
        raise ZeroDivisionError("rotation quaternion has zero norm")
    return np.array([[1.0 - 2 * (y * y + z * z) / n, 2 * (x * y - z * w) / n, 2 * (x * z + y * w) / n],
                     [2 * (x * y + z * w) / n, 1.0 - 2 * (x * x + z * z) / n, 2 * (y * z - x * w) / n],
                     [2 * (x * z - y * w) / n, 2 * (y * z + x * w) / n, 1.0 - 2 * (x * x + y * y) / n]])


def agent_to_world(state):
    """The episode-start agent pose (rotation quaternion, position) as a float64 [4, 4] transform (L655-661)."""
    m = np.eye(4)
    m[:3, :3] = rotation_matrix(state.rotation)
    m[:3, 3] = state.position
    return m


def camera_to_episodic(xyz, yaw, pitch=CAMERA_PITCH):
    """Camera -> episodic frame [4, 4]: yaw about z, then pitch about y, at position xyz, times the axis alignment that
    takes the camera's (right, down, forward) axes to (forward, left, up)."""
    x, y, z = xyz
    c, s, cp, sp = np.cos(yaw), np.sin(yaw), np.cos(pitch), np.sin(pitch)
    yaw_m = np.array([[c, -s, 0, x], [s, c, 0, y], [0, 0, 1, z], [0, 0, 0, 1]])[:3, :3]
    pitch_m = np.array([[cp, 0, sp, x], [0, 1, 0, y], [-sp, 0, cp, z], [0, 0, 0, 1]])[:3, :3]
    m = np.eye(4)
    m[:3, :3] = yaw_m @ pitch_m
    m[:3, 3] = xyz
    return m @ AXIS_ALIGN


def pixel_to_gps(pixel, depth, intrinsic, tf_camera_to_episodic):
    """Image point pixel = (v, u) with depth[v, u] metres -> its (x, y) in the episodic frame.  A point outside the
    depth frame raises IndexError."""
    v, u = pixel
    z = depth[v, u]
    p = np.array([(u - intrinsic[0, 2]) * z / intrinsic[0, 0], (v - intrinsic[1, 2]) * z / intrinsic[1, 1], z, 1.0])
    p = tf_camera_to_episodic @ p
    p = p[:3] / p[3]
    return p[0], p[1]


def follower_action(a):
    """A ShortestPathFollower answer (tensor, array or int) as the action the loop steps (L831-832)."""
    if isinstance(a, torch.Tensor):
        a = a.detach().cpu().numpy()[0]
    return a[0] if hasattr(a, "__len__") else a


def _shortest_path_follower(env):
    from habitat.tasks.nav.shortest_path_follower import ShortestPathFollower
    return ShortestPathFollower(env._env.sim, FOLLOWER_RADIUS, False)


class _Request:
    """What one environment waits for: System 2 ("s2": frame, look_down, instruction, conjunction) or System 1 ("s1":
    the look-down frame and its raw depth, `goal` when this frame becomes the pixel-goal frame)."""
    __slots__ = ("kind", "rgb", "depth", "look_down", "instruction", "conjunction", "goal")

    def __init__(self, kind, rgb, depth=None, look_down=False, instruction=None, conjunction=None, goal=False):
        self.kind, self.rgb, self.depth, self.look_down = kind, rgb, depth, look_down
        self.instruction, self.conjunction, self.goal = instruction, conjunction, goal


class _Env:
    """Driver-side state of one environment: its conjunction draws, the frames that entered its history since the last
    policy call, whether its policy state must be reset first, its latent plan, its results."""

    def __init__(self, seed):
        self.rng = random.Random(seed)
        self.history, self.reset = [], False
        self.latent = None
        self.results = []


class HabitatVLNEvaluator:
    def __init__(self, model, processor, num_history=8, resize_w=384, resize_h=384, min_depth=0.0, max_depth=10.0,
                 max_steps_per_episode=500, depth_filter=None, vision_cache_frames=0, seeds=None, x_init=None,
                 max_new_tokens=128, mode="dual_system", camera_height=None, width=640, height=480, hfov=79,
                 make_follower=None, kv_pool_tokens=None):
        """`depth_filter(depth [H, W], blur_type=None)`: the filter the reference applies to every depth frame; needed
        by a System 1 that reads depth and by the system2 mode.  `seeds`: one `random.Random` seed per environment for
        the conjunction draws, as many as `run_*` gets environments (default 0, 1, ...).  `x_init`: None (System 1 draws its noise on the device) or a callable env_ids ->
        initial noise [len(env_ids) * 32, T, 3] for those environments, in that order.  `max_new_tokens`: System 2's
        answer budget (the reference's 128).

        `mode`: the reference's `model_settings["mode"]`.  "dual_system" (`run_dual_system`) needs a model with a
        System 1; "system2" (`run_system2`) takes any model with `generate` and also needs the sensor geometry --
        `camera_height` (metres, the RGB sensor's position[1] in the caller's habitat config; no default), the RGB
        sensor's `width` x `height` and `hfov` (degrees; vln_r2r.yaml: 640 x 480, 79) and `min_depth` / `max_depth` --
        and `make_follower(env)`, the per-episode ShortestPathFollower (default: habitat's
        `ShortestPathFollower(env._env.sim, 0.25, False)`, imported when first needed)."""
        if mode not in ("dual_system", "system2"):
            raise ValueError("mode must be 'dual_system' or 'system2', not %r" % (mode,))
        if mode == "dual_system" and not getattr(model, "has_system1", True):
            raise ValueError("the dual-system evaluation needs a model with a System 1; this one has none")
        if mode == "system2":
            if not callable(getattr(model, "generate", None)):
                raise ValueError("the system2 evaluation needs a model with generate")
            if camera_height is None:
                raise ValueError("the system2 evaluation needs camera_height: the RGB sensor's height in the habitat "
                                 "config")
            if depth_filter is None:
                raise ValueError("the system2 evaluation needs depth_filter for the depth of pixel answers")
        self.mode = mode
        processor.tokenizer.padding_side = "left"
        self.model, self.processor = model, processor
        self.num_history, self.resize_w, self.resize_h = num_history, resize_w, resize_h
        self.min_depth, self.max_depth = min_depth, max_depth
        self.max_steps_per_episode = max_steps_per_episode
        self.depth_filter, self.vision_cache_frames = depth_filter, vision_cache_frames
        self.kv_pool_tokens = kv_pool_tokens  # see InternVLAN1Policy
        self.seeds, self.max_new_tokens = seeds, max_new_tokens
        self.device = torch.device(getattr(model, "device", "cpu"))
        self.reads_depth = mode == "dual_system" and \
            getattr(getattr(model, "config", None), "system1", None) == "navdp_async"
        if self.reads_depth and depth_filter is None:
            raise ValueError("a System 1 that reads depth (navdp_async) needs depth_filter")
        self.camera_height = camera_height
        self.intrinsic = intrinsic_matrix(width, height, hfov)
        self.make_follower = _shortest_path_follower if make_follower is None else make_follower
        self._frames = self.s1 = None
        if mode == "dual_system":
            self._frames = FramePreprocessor(self.device) if self.device.type == "cuda" else None
            self.s1 = System1Inputs(model, self._frames, x_init)
        self.policy = None
        self.calls = {"s2": 0, "s1": 0, "rounds": 0}

    # ------------------------------------------------------------------ driver
    def run_dual_system(self, envs):
        """Run every episode of every environment -> per environment the list of its episodes' result dicts."""
        return self._run("dual_system", envs, self._episodes)

    def run_system2(self, envs):
        """The system2 mode: run every episode of every environment -> per environment its episodes' result dicts."""
        return self._run("system2", envs, self._episodes_system2)

    def _run(self, mode, envs, episodes):
        if mode != self.mode:
            raise ValueError("run_%s needs an evaluator built with mode=%r; this one has mode=%r" % (mode, mode, self.mode))
        B = len(envs)
        if self.policy is None or len(self.policy.episodes) != B:
            self.policy = P.InternVLAN1Policy(self.model, self.processor, num_envs=B, num_history=self.num_history,
                                              resize_w=self.resize_w, resize_h=self.resize_h,
                                              max_new_tokens=self.max_new_tokens, device=self.device,
                                              vision_cache_frames=self.vision_cache_frames,
                                              system2_only=mode == "system2", kv_pool_tokens=self.kv_pool_tokens)
        self.policy.reset()
        seeds = list(range(B)) if self.seeds is None else list(self.seeds)
        if len(seeds) != B:
            raise ValueError("%d seeds for %d environments: give one seed per environment" % (len(seeds), B))
        state = [_Env(s) for s in seeds]
        gens = [episodes(env, st, e) for e, (env, st) in enumerate(zip(envs, state))]
        req = {}
        for e, g in enumerate(gens):
            self._advance(req, e, g, None)
        while req:
            self._round(req, gens, state)
        return [st.results for st in state]

    def _round(self, req, gens, state):
        """One System-2 call for every environment waiting for System 2, then one System-1 call for every environment
        waiting for System 1 (including those whose System-2 answer was a pixel goal)."""
        self.calls["rounds"] += 1
        s2 = [e for e in sorted(req) if req[e].kind == "s2"]
        if s2:
            self._flush_history(state)
            res = self.policy.s2_step(s2, [req[e].rgb for e in s2], [None] * len(s2), [None] * len(s2),
                                      [req[e].instruction for e in s2], None, [req[e].look_down for e in s2],
                                      conjunctions=[req[e].conjunction for e in s2])
            self.calls["s2"] += 1
            for e, r in zip(s2, res):
                if not isinstance(r, Exception) and r.output_latent is not None:
                    state[e].latent = r.output_latent
                self._advance(req, e, gens[e], r)
        s1 = [e for e in sorted(req) if req[e].kind == "s1"]
        if s1:
            for e, ids in zip(s1, self._system1(s1, [req[e] for e in s1], state)):
                self._advance(req, e, gens[e], ids)

    @staticmethod
    def _advance(req, e, gen, value):
        """Resume environment e's generator with `value` until its next request (or the end of its episodes)."""
        try:
            req[e] = gen.send(value)
        except StopIteration:
            req.pop(e, None)

    def _flush_history(self, state):
        """Policy resets of the environments that started a new episode, then every frame that entered a history since
        the last policy call, in one step_no_infer (an environment may add several)."""
        resets = [e for e, st in enumerate(state) if st.reset]
        if resets:
            self.policy.reset(resets)
        ids = [e for e, st in enumerate(state) for _ in st.history]
        frames = [f for st in state for f in st.history]
        for st in state:
            st.history, st.reset = [], False
        if ids:
            self.policy.step_no_infer(ids, frames)

    # ------------------------------------------------------------------ System 1
    def _system1(self, envs, reqs, state):
        """One generate_traj call for the listed environments -> each one's local action chunk (MAX_LOCAL_STEPS ids)."""
        cur = self.s1.rgb([r.rgb for r in reqs]).to(torch.bfloat16)
        cur_d = None
        if self.reads_depth:
            cur_d = torch.stack([self.s1_depth(r.depth) for r in reqs]).to(self.device)
        traj = self.s1.generate(envs, {e for e, r in zip(envs, reqs) if r.goal}, cur, cur_d,
                                [state[e].latent for e in envs])
        self.calls["s1"] += 1
        lists = batched_traj_to_actions(traj, len(envs), max_actions=MAX_LOCAL_STEPS)
        return [(list(a) + [STOP] * MAX_LOCAL_STEPS)[:MAX_LOCAL_STEPS] for a in lists]

    def s1_depth(self, depth):
        """One raw depth observation ([H, W] or [H, W, 1], normalised) -> host bf16 [224, 224]: the reference's filter,
        affine, `* 1000`, uint16, Pillow I;16 NEAREST resize, `/ 1000`, float32 and clip at 5 (L354-365), with
        everything after the filter computed on the 224 x 224 sampled pixels only."""
        d = np.asarray(depth)
        d = self.depth_filter(d.reshape(d.shape[:2]), blur_type=None)
        d = d[np.ix_(nearest_index(d.shape[0], S1_SIZE), nearest_index(d.shape[1], S1_SIZE))]
        d = d * (self.max_depth - self.min_depth) + self.min_depth
        d = d * 1000
        t = torch.as_tensor(np.ascontiguousarray(d.astype(np.uint16) / 1000)).float()
        t[t > SYS1_DEPTH_THRESHOLD] = SYS1_DEPTH_THRESHOLD
        return t.to(torch.bfloat16)

    # ------------------------------------------------------------------ one environment (L271-606)
    def _episodes(self, env, st, e):
        """The reference loop for one environment; yields a _Request where the reference calls the model and receives
        the S2Output (or Exception) of System 2, or the local action chunk of System 1."""
        while env.is_running:
            obs = env.reset()
            if not env.is_running or obs is None:
                break
            st.history, st.reset, st.latent = [], True, None
            self.s1.reset([e])
            episode = env.get_current_episode()
            scene_id, episode_id = episode.scene_id.split("/")[-2], int(episode.episode_id)
            instruction = episode.instruction.instruction_text
            step_id, action_seq, local_actions, action, pixel_goal, forward_action = 0, [], [], None, None, 0
            done, error = False, None
            while not done and step_id <= self.max_steps_per_episode:
                # frames are copied before the next env.step, where the reference converts them (L326-330, L352-356):
                # a simulator may render every observation into the same buffer
                rgb, depth = self._own(obs)
                look_down_rgb, look_down_depth = rgb, depth
                ask = len(action_seq) == 0 and pixel_goal is None
                if action != LOOKDOWN:
                    if not ask:
                        st.history.append(rgb)   # a System-2 call adds its own frame to the history
                    env.step(LOOKDOWN)
                    down, _, _, _ = env.step(LOOKDOWN)
                    look_down_rgb, look_down_depth = self._own(down)
                    env.step(LOOKUP)
                    env.step(LOOKUP)
                if ask:
                    look_down = action == LOOKDOWN
                    res = yield _Request("s2", rgb, look_down=look_down, instruction=instruction[:-1],
                                         conjunction=st.rng.choice(CONJUNCTIONS))
                    if isinstance(res, Exception):
                        error = res
                        break
                    if res.output_pixel is not None:
                        forward_action, pixel_goal = 0, [int(v) for v in res.output_pixel]
                        env.step(LOOKUP)
                        env.step(LOOKUP)
                        local_actions = yield _Request("s1", look_down_rgb, look_down_depth, goal=True)
                        action = local_actions[0]
                        if action == STOP:
                            pixel_goal, action = None, LEFT
                            obs, _, done, _ = env.step(action)
                            step_id += 1
                            continue
                    else:
                        action_seq = list(res.output_action)
                if len(action_seq) != 0:
                    action = action_seq.pop(0)
                elif pixel_goal is not None:
                    if len(local_actions) == 0:
                        local_actions = yield _Request("s1", look_down_rgb, look_down_depth)
                    action = local_actions.pop(0)
                    forward_action += 1
                    if forward_action > MAX_STEPS or action == STOP:
                        pixel_goal, forward_action, local_actions = None, 0, []
                        step_id += 1
                        continue
                else:
                    action = STOP
                if action == LOOKDOWN:
                    env.step(action)
                    obs, _, done, _ = env.step(action)
                else:
                    obs, _, done, _ = env.step(action)
                    step_id += 1
            st.results.append(self._result(env, scene_id, episode_id, step_id, instruction, error))

    @staticmethod
    def _result(env, scene_id, episode_id, step_id, instruction, error):
        """The episode's progress.json dict (L590-601 / L909-920), plus the error that ended it, if any."""
        metrics = env.get_metrics()
        result = {"scene_id": scene_id, "episode_id": episode_id, "success": metrics["success"],
                  "spl": metrics["spl"], "os": metrics["oracle_success"], "ne": metrics["distance_to_goal"],
                  "steps": step_id, "episode_instruction": instruction}
        if "ndtw" in metrics:
            result["ndtw"] = metrics["ndtw"]
        if error is not None:
            result["error"], result["error_message"] = type(error).__name__, str(error)
        return result

    def _own(self, obs):
        """Copies of an observation's RGB frame and, for a System 1 that reads depth, its depth frame (else None)."""
        return np.array(obs["rgb"]), (np.array(obs["depth"]) if self.reads_depth else None)

    # ------------------------------------------------------------------ one environment, system2 mode (L640-935)
    def _episodes_system2(self, env, st, e):
        """The reference's system2 loop for environment e; yields a _Request where the reference calls the model and
        receives the S2Output (or Exception) of System 2."""
        while env.is_running:
            obs = env.reset()
            if not env.is_running or obs is None:
                break
            st.history, st.reset = [], True
            episode = env.get_current_episode()
            scene_id, episode_id = episode.scene_id.split("/")[-2], int(episode.episode_id)
            instruction = episode.instruction.instruction_text
            sim = env._env.sim
            to_world = agent_to_world(sim.get_agent_state())
            follower = self.make_follower(env)
            initial_height = sim.get_agent_state().position[1]
            step_id, action_seq, action, goal, forward_action = 0, [], None, None, 0
            talking = False     # the last System-2 conversation is still open: no action step since
            done, error = False, None
            # the observation is copied when it arrives: an iteration that takes no step shows the same one again
            cur = self._own_system2(obs)
            while not done and step_id <= self.max_steps_per_episode:
                rgb, depth, gps, compass = cur
                ask = len(action_seq) == 0 and goal is None
                if action != LOOKDOWN and not ask:
                    st.history.append(rgb)   # a System-2 call adds its own frame to the history
                if ask:
                    height = sim.get_agent_state().position[1] - initial_height
                    look_down = action == LOOKDOWN
                    conjunction = st.rng.choice(CONJUNCTIONS)
                    if look_down and not talking:
                        n = len(self.policy.episodes[e].input_images) + 1
                        error = ValueError("a look-down turn after an action step: the cleared conversation has 1 image "
                                           "placeholder for %d images" % n)
                        break
                    res = yield _Request("s2", rgb, look_down=look_down, instruction=instruction[:-1],
                                         conjunction=conjunction)
                    if isinstance(res, Exception):
                        error = res
                        break
                    talking = True
                    if res.output_pixel is not None:
                        forward_action = 0
                        env.step(LOOKUP)
                        env.step(LOOKUP)
                        try:
                            goal = self._world_goal(sim, [int(v) for v in res.output_pixel], depth, gps, compass,
                                                    height, to_world)
                        except IndexError as exc:
                            error = exc
                            break
                        if follower.get_next_action(goal) == STOP:
                            goal, action, talking = None, LEFT, False
                            obs, _, done, _ = env.step(action)
                            cur = self._own_system2(obs)
                            step_id += 1
                            continue
                    else:
                        action_seq = list(res.output_action)
                if len(action_seq) != 0:
                    action = action_seq.pop(0)
                elif goal is not None:
                    action = follower_action(follower.get_next_action(goal))
                    forward_action += 1
                    if forward_action > MAX_STEPS or action == STOP:
                        goal, forward_action, talking = None, 0, False
                        step_id += 1
                        continue
                else:
                    action = STOP
                if action == LOOKDOWN:
                    env.step(action)
                    obs, _, done, _ = env.step(action)
                else:
                    obs, _, done, _ = env.step(action)
                    step_id += 1
                    talking = False
                cur = self._own_system2(obs)
            st.results.append(self._result(env, scene_id, episode_id, step_id, instruction, error))

    def _world_goal(self, sim, pixel, depth, gps, compass, height, to_world):
        """A pixel answer -> its navigable world goal (L710-712, L716-719, L804-809): the depth frame filtered, scaled
        to metres and lifted through the camera pose of this iteration, then taken to the world frame by the
        episode-start agent pose and snapped to the navmesh unless navigable."""
        d = self.depth_filter(depth.reshape(depth.shape[:2]), blur_type=None)
        d = d * (self.max_depth - self.min_depth) + self.min_depth
        d = d * 1000
        x, y = gps
        tf = camera_to_episodic(np.array([x, -y, self.camera_height + height]), compass[0])
        g = pixel_to_gps(pixel, d / 1000, self.intrinsic, tf)
        goal = (to_world @ np.array([-g[1], 0, -g[0], 1]))[:3]
        if not sim.pathfinder.is_navigable(np.array(goal)):
            goal = np.array(sim.pathfinder.snap_point(np.array(goal)))
        return goal

    @staticmethod
    def _own_system2(obs):
        """Copies of an observation's RGB, depth, gps and compass."""
        return np.array(obs["rgb"]), np.array(obs["depth"]), np.array(obs["gps"]), np.array(obs["compass"])
