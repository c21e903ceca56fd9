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
`InternVLAN1Policy`.  On a CUDA device the System-1 RGB frames of a round are uploaded and resized in one
`FramePreprocessor.rgb` call and cast to bf16: the kernel's float32 u / 255 rounded to bf16 is torch's
`bf16(u8) / 255` for every byte.  Each environment keeps its pixel-goal frame on the device.  Depth is prepared only for
a System 1 that reads it (`navdp_async`): `depth_filter` runs on the full frame on the host, as in the reference; then
only the 224 x 224 source pixels of Pillow's NEAREST resize are taken (`nearest_index`) and the affine, `* 1000`, the
uint16 truncation, `/ 1000`, float32, the clip at 5 and bf16 are applied to those samples.  Every step after the filter
is element-wise, so this is the reference's full-frame path bit for bit.  On the CPU the frames go through Pillow.

Deviations from the reference loop:
  * nothing is written (no check_sim images, videos, progress.json or resume) and nothing is printed; the caller
    writes the returned dicts;
  * a look-down turn continues its conversation on the K/V cache (byte-identical output, see InternVLAN1Policy);
  * the pixel goal's latent plan comes from the generate pass's cache instead of a second prefill (`generate_with_latents`);
  * an answer the reference cannot parse (a lone number: IndexError at L436, which ends the reference's run) ends that
    environment's episode; its dict holds `get_metrics()` at that point, the exception's type name under "error" and its
    message under "error_message" (so every dict stays JSON-serialisable), and the other environments carry on;
  * `depth_filter` is supplied by the caller (the reference calls `depth_camera_filtering.filter_depth`).
The evaluator's `system2` mode needs the simulator's ShortestPathFollower and is not mirrored.
"""
import random

import numpy as np
import torch
from PIL import Image

from . import policy as P
from .agent_realworld import InternVLAN1AsyncAgent
from .postprocess import batched_traj_to_actions

S1_SIZE = 224
MAX_STEPS, MAX_LOCAL_STEPS = 8, 4
STOP, FORWARD, LEFT, RIGHT, LOOKUP, LOOKDOWN = range(6)
DEPTH_CLIP = 5.0
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


class _Request:
    """What one environment waits for: System 2 ("s2": frame, look_down, instruction, conjunction) or System 1 ("s1":
    the look-down frame and its raw depth, `goal` when this frame becomes the pixel-goal frame)."""
    __slots__ = ("kind", "rgb", "depth", "look_down", "instruction", "conjunction", "goal")

    def __init__(self, kind, rgb, depth=None, look_down=False, instruction=None, conjunction=None, goal=False):
        self.kind, self.rgb, self.depth, self.look_down = kind, rgb, depth, look_down
        self.instruction, self.conjunction, self.goal = instruction, conjunction, goal


class _Env:
    """Driver-side state of one environment: its conjunction draws, the frames that entered its history since the last
    policy call, whether its policy state must be reset first, its pixel-goal frames and latent plan, its results."""

    def __init__(self, seed):
        self.rng = random.Random(seed)
        self.history, self.reset = [], False
        self.goal_rgb = self.goal_depth = self.latent = None
        self.results = []


class HabitatVLNEvaluator:
    def __init__(self, model, processor, num_history=8, resize_w=384, resize_h=384, min_depth=0.0, max_depth=10.0,
                 max_steps_per_episode=500, depth_filter=None, vision_cache_frames=0, seeds=None, x_init=None,
                 max_new_tokens=128):
        """`depth_filter(depth [H, W], blur_type=None)`: the filter the reference applies to every depth frame; needed
        only by a System 1 that reads depth.  `seeds`: one `random.Random` seed per environment for the conjunction
        draws, as many as `run_dual_system` gets environments (default 0, 1, ...).  `x_init`: None (System 1 draws its noise on the device) or a callable env_ids ->
        initial noise [len(env_ids) * 32, T, 3] for those environments, in that order.  `max_new_tokens`: System 2's
        answer budget (the reference's 128)."""
        if not getattr(model, "has_system1", True):
            raise ValueError("the dual-system evaluation needs a model with a System 1; this one has none")
        processor.tokenizer.padding_side = "left"
        self.model, self.processor = model, processor
        self.num_history, self.resize_w, self.resize_h = num_history, resize_w, resize_h
        self.min_depth, self.max_depth = min_depth, max_depth
        self.max_steps_per_episode = max_steps_per_episode
        self.depth_filter, self.vision_cache_frames = depth_filter, vision_cache_frames
        self.seeds, self.x_init, self.max_new_tokens = seeds, x_init, max_new_tokens
        self.device = torch.device(getattr(model, "device", "cpu"))
        self.reads_depth = getattr(getattr(model, "config", None), "system1", None) == "navdp_async"
        if self.reads_depth and depth_filter is None:
            raise ValueError("a System 1 that reads depth (navdp_async) needs depth_filter")
        self._frames = None
        if self.device.type == "cuda":
            from .preprocess import FramePreprocessor
            self._frames = FramePreprocessor(self.device, out_size=S1_SIZE)
        self.policy = None
        self.calls = {"s2": 0, "s1": 0, "rounds": 0}

    # ------------------------------------------------------------------ driver
    def run_dual_system(self, envs):
        """Run every episode of every environment -> per environment the list of its episodes' result dicts."""
        B = len(envs)
        if self.policy is None or len(self.policy.episodes) != B:
            self.policy = P.InternVLAN1Policy(self.model, self.processor, num_envs=B, num_history=self.num_history,
                                              resize_w=self.resize_w, resize_h=self.resize_h,
                                              max_new_tokens=self.max_new_tokens, device=self.device,
                                              vision_cache_frames=self.vision_cache_frames)
        self.policy.reset()
        seeds = list(range(B)) if self.seeds is None else list(self.seeds)
        if len(seeds) != B:
            raise ValueError("%d seeds for %d environments: give one seed per environment" % (len(seeds), B))
        state = [_Env(s) for s in seeds]
        gens = [self._episodes(env, st) for env, st in zip(envs, state)]
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
        cur = self._rgb224([r.rgb for r in reqs])
        cur_d = None
        if self.reads_depth:
            cur_d = torch.stack([self.s1_depth(r.depth) for r in reqs]).to(self.device)
        for k, (e, r) in enumerate(zip(envs, reqs)):
            if r.goal:
                state[e].goal_rgb = cur[k].clone()
                state[e].goal_depth = None if cur_d is None else cur_d[k].clone()
        rgb = torch.stack([torch.stack((state[e].goal_rgb, cur[k])) for k, e in enumerate(envs)])
        dep = None
        if cur_d is not None:
            dep = torch.stack([torch.stack((state[e].goal_depth, cur_d[k])) for k, e in enumerate(envs)])[..., None]
        lat = torch.cat([state[e].latent.reshape(1, *state[e].latent.shape[-2:]) for e in envs])
        kw = {} if self.x_init is None else {"x_init": self.x_init(envs)}
        with torch.no_grad():
            traj = self.model.generate_traj(lat, rgb, dep, **kw)
        self.calls["s1"] += 1
        lists = batched_traj_to_actions(traj, len(envs), max_actions=MAX_LOCAL_STEPS)
        return [(list(a) + [STOP] * MAX_LOCAL_STEPS)[:MAX_LOCAL_STEPS] for a in lists]

    def _rgb224(self, frames):
        """Raw uint8 look-down frames -> bf16 [n, 224, 224, 3] = bf16(Pillow-resized u8) / 255, on the device."""
        if self._frames is None:
            u8 = np.stack([np.array(Image.fromarray(np.asarray(f)).convert("RGB").resize((S1_SIZE, S1_SIZE)))
                           for f in frames])
            return torch.from_numpy(u8).to(torch.bfloat16) / 255
        return InternVLAN1AsyncAgent._by_shape(frames, self._frames.rgb).to(torch.bfloat16)

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
        t[t > DEPTH_CLIP] = DEPTH_CLIP
        return t.to(torch.bfloat16)

    # ------------------------------------------------------------------ one environment (L271-606)
    def _episodes(self, env, st):
        """The reference loop for one environment; yields a _Request where the reference calls the model and receives
        the S2Output (or Exception) of System 2, or the local action chunk of System 1."""
        while env.is_running:
            obs = env.reset()
            if not env.is_running or obs is None:
                break
            st.history, st.reset, st.goal_rgb, st.goal_depth, st.latent = [], True, None, None, None
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
            metrics = env.get_metrics()
            result = {"scene_id": scene_id, "episode_id": episode_id, "success": metrics["success"],
                      "spl": metrics["spl"], "os": metrics["oracle_success"], "ne": metrics["distance_to_goal"],
                      "steps": step_id, "episode_instruction": instruction}
            if "ndtw" in metrics:
                result["ndtw"] = metrics["ndtw"]
            if error is not None:
                result["error"], result["error_message"] = type(error).__name__, str(error)
            st.results.append(result)

    def _own(self, obs):
        """Copies of an observation's RGB frame and, for a System 1 that reads depth, its depth frame (else None)."""
        return np.array(obs["rgb"]), (np.array(obs["depth"]) if self.reads_depth else None)
