"""Batched VL-LN dialog / ObjectNav evaluation: the episode loop of the Habitat dialog evaluator for B environments at once.

Mirrors `HabitatDialogEvaluator.eval_action` / `calc_metrics` (internnav/habitat_extensions/vlln/habitat_dialog_evaluator.py
L93-273) and the agent it drives, `DialogAgent` (internnav/agent/dialog_agent.py L131-338), the loop behind the
reference's VL-LN instance-dialog and HM3D ObjectNav numbers, which runs one environment per process and one System-2
`generate` per turn.  Per environment the loop is the reference's, transcribed as a generator (`_episodes`) that yields
wherever the reference calls System 2 or the oracle NPC:

  * the instruction is "search for {category}., " + the instruction (`coin`), "search for {category}." (`objectnav`), or
    the instruction without its last character (L116-127);
  * every call but a look-down or dialog turn adds the (resized) frame to the history, a look-down turn keeps its frame
    at full size (L151-157); an action 7 does not update the last action, so the next call adds the same frame again;
  * System 2 is asked when no action and no goal is held (L298).  A fresh turn builds the user message from the prompt
    (with the oracle sentence for a dialog task or `dialog_enabled`), the history ids `unique(linspace(0, step_id - 1,
    num_history))` merged with the steps of earlier dialogs, each dialog's text after its history image, the previous
    look-down image (`append_look_down`) and the current frame; a look-down turn appends the full-size frame and the
    previous answer; a dialog turn records question and answer in `dialogs` and appends the question and the NPC's
    answer as text, with no image (L211-277).  The conjunction is drawn from the environment's `random.Random`;
  * an answer with "<talk>" is a question (action 6); else one with a digit is a pixel goal: a lone number or a point
    outside the depth frame is action 0; the goal is lifted through the filtered depth (`* 1000`, `/ 1000`) and a 30
    degree camera pose, taken to the world frame by the episode-start pose and snapped unless navigable; the camera
    steps LOOKUP twice, the previous look-down image is updated, and a follower answer of 0 turns into action 2 with
    the goal dropped (L160-209); anything else is an action list;
  * with a goal the follower is asked once per step; more than 8 calls or a STOP drop the goal and return 7 (L310-331);
  * action 5 steps twice, 6 asks the NPC (past `turn` questions the answer is the fixed question-limit text, a None
    answer becomes "Sorry, I can not answer your question now."), 5 / 6 / 7 do not count a step, 0-3 step and clear the
    conversation, and an episode runs while it is not over and step_id <= max_steps_per_episode (L156-209).

`run(envs)` drives B such generators in rounds.  A round serves every environment waiting for System 2 -- fresh,
look-down and dialog turns alike -- in ONE `DialogPolicy.s2_step` (one `generate`), then every question to the oracle
in ONE call of the caller's `npc`.  A dialog turn continues its conversation on the environment's K/V slot: only the
question and the NPC's answer are prefilled and the vision tower does not run.

Deviations from the reference loop:
  * nothing is written (check_sim images, action logs, videos, progress.json, resume) and nothing is printed; the caller
    writes the returned dicts;
  * look-down and dialog turns continue their conversation on the K/V cache (byte-identical output);
  * depth is filtered only for pixel answers (the reference filters every frame; the goals are the same);
  * the NPC is the caller's `npc` callable, which stands for `get_description` + `SimpleNPC.answer_question`;
  * two failures end only that environment's episode, with `error` / `error_message` (the reference's run ends): a
    look-down or dialog turn whose conversation has been cleared -- by an action step of the same answer ("←↓"), or by
    a follower stop (action 7) after a question, which leaves the last action at 6 -- so that the chat has one image
    placeholder or none for all of the conversation's images, which Qwen2.5-VL refuses; and a question in an
    evaluator without `npc` (the reference reads scene files it loads only for dialog tasks).
"""
import random
import re

import numpy as np
import torch
from PIL import Image

from . import policy as P
from .agent import intrinsic_matrix
from .habitat_eval import (CONJUNCTIONS, MAX_STEPS, agent_to_world, camera_to_episodic, follower_action, pixel_to_gps,
                           summarize, _shortest_path_follower)

STOP, FORWARD, LEFT, RIGHT, LOOKUP, LOOKDOWN, TALK, NOOP = range(8)
PROMPT_DIALOG = (
    "You are an autonomous navigation assistant. Your task is to <instruction>. Where should you go next to stay on "
    "track? There is an oracle can help you to complete the task in current environment, you can either choose to move "
    "or talk. If choosing to talk, please say something that can help you better to find the target object. If choosing "
    "to move, when you want to output a waypoint you need to TILT DOWN (↓) by 30 degrees then output the next "
    "waypoint\'s coordinates in the image. In case the next waypoint is out of view, utilize the turn actions: TURN LEFT "
    "(←) or TURN RIGHT (→) by 15 degrees. Please output STOP when you have successfully completed the task.")
PROMPT_NAVIGATE = (
    "You are an autonomous navigation assistant. Your task is to <instruction>. Where should you go next to stay on "
    "track? When you want to output a waypoint you need to TILT DOWN (↓) by 30 degrees then output the next waypoint\'s "
    "coordinates in the image. In case the next waypoint is out of view, utilize the turn actions: TURN LEFT (←) or TURN "
    "RIGHT (→) by 15 degrees. Please output STOP when you have successfully completed the task.")
QUESTION_LIMIT = "Sorry, you have reached the question limit. No further answers are available."
NO_ANSWER = "Sorry, I can not answer your question now."
OBJECTNAV_INSTRUCTION = "search for {target_object}."
CLEARED = "a turn that continues a cleared conversation has %d image placeholders for %d images"


def summarize_dialog(results):
    """`calc_metrics` (L251-273) over per-episode result dicts: float32 means of success, SPL (NaN / inf count as 0),
    oracle success and the finite navigation errors -> {sucs_all, spls_all, oss_all, nes_all}."""
    return summarize([{k: r[k] for k in ("success", "spl", "os", "ne")} for r in results])


class _Turn:
    """One System-2 turn of one environment: "fresh", "look_down" or "dialog", the instruction, the step id, and for a
    dialog turn the NPC's answer."""
    __slots__ = ("kind", "instruction", "step_id", "npc_answer")

    def __init__(self, kind, instruction, step_id, npc_answer=None):
        self.kind, self.instruction, self.step_id, self.npc_answer = kind, instruction, step_id, npc_answer


class _DialogEpisode(P._Episode):
    """The dialog agent's conversation state (L340-360): the policy's, plus the previous look-down image and the dialogs."""

    def __init__(self):
        super().__init__()
        self.prev_look_image = None
        self.dialogs = []


class DialogPolicy(P.InternVLAN1Policy):
    """`InternVLAN1Policy` with the dialog agent's conversation (`_chat`, L211-277): the device frame path, the K/V and
    feature pools and the single `generate` call of `s2_step` are the base class's.  `s2_step` takes a `_Turn` per
    environment in place of the instruction, the turn's new frame (the full-size look-down frame, or None: a fresh
    turn's frame is already the history's last, a dialog turn brings none) and `continues` in place of `look_downs`,
    and returns each environment's answer text (or the Exception its preparation raised).  Frames enter the history
    through `step_no_infer`, as the reference's `convert_input` adds them."""

    def __init__(self, model, processor, num_envs=1, num_history=8, resize_w=384, resize_h=384, max_new_tokens=128,
                 device=None, vision_cache_frames=0, prompt=PROMPT_DIALOG, append_look_down=False, turn=5,
                 frame_shape=(480, 640), npc_tokens=128, kv_pool_tokens=None):
        super().__init__(model, processor, num_envs=num_envs, num_history=num_history, resize_w=resize_w,
                         resize_h=resize_h, max_new_tokens=max_new_tokens, device=device,
                         vision_cache_frames=vision_cache_frames, system2_only=True, kv_pool_tokens=kv_pool_tokens)
        self.episodes = [_DialogEpisode() for _ in range(num_envs)]
        self.prompt, self.append_look_down, self.turn = prompt, append_look_down, int(turn)
        self.frame_shape, self.npc_tokens = tuple(frame_shape), int(npc_tokens)

    def reset(self, env_ids=None):
        super().reset(env_ids)
        for e in (range(len(self.episodes)) if env_ids is None else env_ids):
            self.episodes[e] = _DialogEpisode()

    def _frame_shape(self, rgbs):
        return self.frame_shape

    def _kv_capacity(self, frame_h, frame_w):
        """Tokens one environment's slot must hold.  A fresh turn carries up to num_history + turn + 2 resized frames
        (the history, the steps of earlier dialogs, the previous look-down image and the current frame) and the
        conversation may add the full-size look-down frame, so with F the tokens of a resized frame and F_full those of
        a full-size one:

            (num_history + turn + 2) F + F_full + (turn + 2) max_new_tokens + turn npc_tokens
              + turn (max_new_tokens + npc_tokens) + 512

        -- up to turn + 2 answers (questions, the answer before a look-down turn, the last answer), `turn` NPC answers
        of `npc_tokens`, the text of up to `turn` earlier dialogs in the history prompt, and 512 tokens of prompt text.
        A conversation that still does not fit (questions past the turn limit, long answers) runs uncached."""
        frame, full = P._image_tokens(self.resize_h, self.resize_w), P._image_tokens(frame_h, frame_w)
        return ((self.num_history + self.turn + 2) * frame + full + (self.turn + 2) * self.max_new_tokens +
                self.turn * self.npc_tokens + self.turn * (self.max_new_tokens + self.npc_tokens) + 512)

    def _feature_rows(self, frame_h, frame_w):
        """Rows of the vision-feature pool: vision_cache_frames resized frames per environment, plus the most one call
        can need at once (every environment's fresh-turn images, num_history + turn + 2 resized frames, and a
        full-size look-down frame)."""
        n, frame = len(self.episodes), P._image_tokens(self.resize_h, self.resize_w)
        return n * self.vision_cache_frames * frame + n * ((self.num_history + self.turn + 2) * frame +
                                                           P._image_tokens(frame_h, frame_w))

    def set_prev_look(self, env_id, rgb):
        """The previous look-down image of environment env_id becomes raw frame `rgb`, resized (L197-198)."""
        if self._vl is not None:
            image = self._device_frames([rgb], [True])[0]
        else:
            image = Image.fromarray(rgb).convert("RGB").resize((self.resize_w, self.resize_h))
        self.episodes[env_id].prev_look_image = image

    def clear_conversation(self, env_id):
        self.episodes[env_id].conversation_history = []

    def _chat(self, ep, image, turn, continues, conjunction=P.CONJUNCTION):
        """L211-279 for one environment -> the chat text, one image placeholder per image of ep.input_images."""
        if turn.kind == "dialog":
            ep.dialogs.append({"role": "navigator", "message": ep.llm_output.replace("<talk>", ""),
                               "true_idx": turn.step_id})
            ep.dialogs.append({"role": "oracle", "message": turn.npc_answer, "true_idx": turn.step_id})
            ep.conversation_history.append({"role": "assistant", "content": [{"type": "text", "text": ep.llm_output}]})
            ep.conversation_history.append({"role": "user", "content": [{"type": "text", "text": turn.npc_answer}]})
            return self.processor.apply_chat_template(ep.conversation_history, tokenize=False, add_generation_prompt=True)
        if turn.kind == "look_down":
            ep.input_images.append(image)
            ep.conversation_history.append({"role": "assistant", "content": [{"type": "text", "text": ep.llm_output}]})
            text, img_id = "", -1
        else:
            text = self.prompt.replace("<instruction>", turn.instruction)
            history_id = []
            if turn.step_id > 0:
                history_id = np.unique(np.linspace(0, turn.step_id - 1, self.num_history, dtype=np.int32)).tolist()
                dialogs_idx = np.sort(list(set(d["true_idx"] for d in ep.dialogs))).tolist()
                history_id = np.sort(np.unique(np.concatenate([history_id, dialogs_idx]).astype(np.int32))).tolist()
                placeholder = [""] * (len(history_id) + 1)
                for n in dialogs_idx:
                    said = "".join("<|%s|>%s" % (d["role"], d["message"]) for d in ep.dialogs if d["true_idx"] == n)
                    placeholder[history_id.index(n) + 1] = "<|dialog_start|>" + said + "<|dialog_end|>"
                text += " These are your historical observations: %s." % (P.DEFAULT_IMAGE_TOKEN + "\n").join(placeholder)
                if self.append_look_down:
                    text += (" Your previous look down image is:%s." % P.DEFAULT_IMAGE_TOKEN
                             if ep.prev_look_image is not None else " Your previous look down image is not here.")
            look = [ep.prev_look_image] if self.append_look_down and ep.prev_look_image is not None else []
            ep.input_images = [ep.rgb_list[i] for i in sorted(history_id)] + look + ep.rgb_list[-1:]
            img_id = 0
        text += " %s." % (conjunction + P.DEFAULT_IMAGE_TOKEN)
        content = []
        for part in P.split_and_clean(text):
            if part == P.DEFAULT_IMAGE_TOKEN:
                content.append({"type": "image", "image": ep.input_images[img_id]})
                img_id += 1
            else:
                content.append({"type": "text", "text": part})
        ep.conversation_history.append({"role": "user", "content": content})
        return self.processor.apply_chat_template(ep.conversation_history, tokenize=False, add_generation_prompt=True)

    def _answer(self, ep, out, n):
        return ep.llm_output


class _Request:
    """What one environment waits for: System 2 ("s2": its _Turn, the new frame, the conjunction) or the NPC ("npc":
    the observation and the question)."""
    __slots__ = ("kind", "turn", "rgb", "conjunction", "obs", "question")

    def __init__(self, kind, turn=None, rgb=None, conjunction=None, obs=None, question=None):
        self.kind, self.turn, self.rgb, self.conjunction, self.obs, self.question = \
            kind, turn, rgb, conjunction, obs, question


class _Env:
    """Driver-side state of one environment: its conjunction draws, the frames that entered its history since the last
    policy call, its results."""

    def __init__(self, seed):
        self.rng = random.Random(seed)
        self.history, self.results = [], []


class HabitatDialogEvaluator:
    def __init__(self, model, processor, task="instance_dialog", dialog_enabled=False, turn=5, append_look_down=False,
                 num_history=8, resize_w=384, resize_h=384, min_depth=0.0, max_depth=10.0, max_steps_per_episode=500,
                 depth_filter=None, npc=None, make_follower=None, camera_height=None, width=640, height=480, hfov=79,
                 seeds=None, max_new_tokens=128, vision_cache_frames=0, npc_tokens=128, mode="system2",
                 kv_pool_tokens=None):
        """`task`: the task name ("instance_dialog", "objectnav", "coin", ...); the oracle sentence is in the prompt
        when it contains "dialog" or with `dialog_enabled`.  `turn`: questions the NPC answers per episode.
        `npc([(env_index, env, obs, question), ...]) -> [answer str or None, ...]`: the oracle, called once per round
        for every question under the turn limit (the reference's `get_description` + `SimpleNPC.answer_question`).
        `depth_filter(depth [H, W], blur_type=None)`: the reference's `filter_depth`.  `make_follower(env)`: the
        per-episode ShortestPathFollower (default habitat's `ShortestPathFollower(env._env.sim, 0.25, False)`).
        `camera_height` (metres, the RGB sensor's position[1]), `width` x `height`, `hfov` (degrees) and `min_depth` /
        `max_depth`: the sensor geometry.  `seeds`: one conjunction seed per environment (default 0, 1, ...).
        `npc_tokens`: the NPC answer length the K/V slots are sized for."""
        if mode == "dual_system":
            raise NotImplementedError("Dual System mode is not supported in the dialog evaluation")
        if mode != "system2":
            raise ValueError("mode must be 'system2', not %r" % (mode,))
        if not callable(getattr(model, "generate", None)):
            raise ValueError("the dialog evaluation needs a model with generate")
        if camera_height is None:
            raise ValueError("the dialog evaluation needs camera_height: the RGB sensor's height in the habitat config")
        if depth_filter is None:
            raise ValueError("the dialog evaluation needs depth_filter for the depth of pixel answers")
        if npc is not None and not callable(npc):
            raise ValueError("npc must be a callable [(env_index, env, obs, question), ...] -> [answer or None, ...]")
        if int(turn) < 0:
            raise ValueError("turn must be >= 0")
        processor.tokenizer.padding_side = "left"
        self.model, self.processor = model, processor
        self.task, self.turn, self.append_look_down = task, int(turn), bool(append_look_down)
        self.prompt = PROMPT_DIALOG if "dialog" in task or dialog_enabled else PROMPT_NAVIGATE
        self.num_history, self.resize_w, self.resize_h = num_history, resize_w, resize_h
        self.min_depth, self.max_depth = min_depth, max_depth
        self.max_steps_per_episode = max_steps_per_episode
        self.depth_filter, self.npc = depth_filter, npc
        self.make_follower = _shortest_path_follower if make_follower is None else make_follower
        self.camera_height, self.frame_shape = camera_height, (height, width)
        self.intrinsic = intrinsic_matrix(width, height, hfov)
        self.seeds, self.max_new_tokens = seeds, max_new_tokens
        self.vision_cache_frames, self.npc_tokens = vision_cache_frames, npc_tokens
        self.kv_pool_tokens = kv_pool_tokens  # see InternVLAN1Policy
        self.device = torch.device(getattr(model, "device", "cpu"))
        self.policy = None
        self.calls = {"s2": 0, "npc": 0, "rounds": 0}

    # ------------------------------------------------------------------ driver
    def run(self, envs):
        """Run every episode of every environment -> per environment the list of its episodes' result dicts."""
        B = len(envs)
        if self.policy is None or len(self.policy.episodes) != B:
            self.policy = DialogPolicy(self.model, self.processor, num_envs=B, num_history=self.num_history,
                                       resize_w=self.resize_w, resize_h=self.resize_h,
                                       max_new_tokens=self.max_new_tokens, device=self.device,
                                       vision_cache_frames=self.vision_cache_frames, prompt=self.prompt,
                                       append_look_down=self.append_look_down, turn=self.turn,
                                       frame_shape=self.frame_shape, npc_tokens=self.npc_tokens,
                                       kv_pool_tokens=self.kv_pool_tokens)
        self.policy.reset()
        seeds = list(range(B)) if self.seeds is None else list(self.seeds)
        if len(seeds) != B:
            raise ValueError("%d seeds for %d environments: give one seed per environment" % (len(seeds), B))
        state = [_Env(s) for s in seeds]
        gens = [self._episodes(env, st, e) for e, (env, st) in enumerate(zip(envs, state))]
        req = {}
        for e, g in enumerate(gens):
            self._advance(req, e, g, None)
        while req:
            self._round(req, gens, state, envs)
        return [st.results for st in state]

    def _round(self, req, gens, state, envs):
        """One System-2 call for every environment waiting for System 2, then one NPC call for every question."""
        self.calls["rounds"] += 1
        s2 = [e for e in sorted(req) if req[e].kind == "s2"]
        if s2:
            ids = [e for e, st in enumerate(state) for _ in st.history]
            frames = [f for st in state for f in st.history]
            for st in state:
                st.history = []
            if ids:
                self.policy.step_no_infer(ids, frames)
            res = self.policy.s2_step(s2, [req[e].rgb for e in s2], [None] * len(s2), [None] * len(s2),
                                      [req[e].turn for e in s2], None, [req[e].turn.kind != "fresh" for e in s2],
                                      conjunctions=[req[e].conjunction for e in s2])
            self.calls["s2"] += 1
            for e, r in zip(s2, res):
                self._advance(req, e, gens[e], r)
        talk = [e for e in sorted(req) if req[e].kind == "npc"]
        if talk:
            answers = list(self.npc([(e, envs[e], req[e].obs, req[e].question) for e in talk]))
            self.calls["npc"] += 1
            if len(answers) != len(talk):
                raise ValueError("npc answered %d of %d questions" % (len(answers), len(talk)))
            for e, a in zip(talk, answers):
                self._advance(req, e, gens[e], a)

    @staticmethod
    def _advance(req, e, gen, value):
        """Resume environment e's generator with `value` until its next request (or the end of its episodes)."""
        try:
            req[e] = gen.send(value)
        except StopIteration:
            req.pop(e, None)

    def _instruction(self, episode):
        """L116-127."""
        if "coin" in self.task:
            category = OBJECTNAV_INSTRUCTION.format(target_object=episode.object_category.replace("_", " "))
            return category + ", " + episode.instruction
        if "objectnav" in self.task:
            return OBJECTNAV_INSTRUCTION.format(target_object=episode.object_category.replace("_", " "))
        return episode.instruction.instruction_text[:-1]

    # ------------------------------------------------------------------ one environment (L107-241, agent L292-338)
    def _episodes(self, env, st, e):
        """The reference loop for environment e; yields a _Request where the reference calls System 2 (and receives the
        answer text or an Exception) or the NPC (and receives its answer or None)."""
        pol = self.policy
        while env.is_running:
            obs = env.reset()
            if not env.is_running or obs is None:
                break
            episode = env._env.current_episode
            scene_id, episode_id = episode.scene_id.split("/")[-2], int(episode.episode_id)
            instruction = self._instruction(episode)
            # agent.reset (L340-360)
            st.history = []
            pol.reset([e])
            sim = env._env.sim
            follower = self.make_follower(env)
            start = sim.get_agent_state()
            to_world, initial_height = agent_to_world(start), start.position[1]
            last_action, action_seq, goal, forward_action, look_down_rgb = None, [], None, 0, None
            step_id, path, actions, error, npc_answer = 0, [], [], None, None
            cur = self._own(obs)
            while not env._env.episode_over and step_id <= self.max_steps_per_episode:
                state = sim.get_agent_state()
                path.append(state.position.tolist())
                rgb, depth, gps, compass = cur
                # convert_input (L131-158)
                if last_action == LOOKDOWN:
                    look_down_rgb = rgb
                elif last_action != TALK:
                    st.history.append(rgb)
                action = None
                if len(action_seq) == 0 and goal is None:
                    kind = "dialog" if last_action == TALK else ("look_down" if last_action == LOOKDOWN else "fresh")
                    conjunction = None if kind == "dialog" else st.rng.choice(CONJUNCTIONS)
                    ep = pol.episodes[e]
                    if kind != "fresh" and not ep.conversation_history:
                        ld = int(kind == "look_down")
                        error = ValueError(CLEARED % (ld, len(ep.input_images) + ld))
                        break
                    text = yield _Request("s2", _Turn(kind, instruction, step_id, npc_answer),
                                          look_down_rgb if kind == "look_down" else None, conjunction)
                    if isinstance(text, Exception):
                        error = text
                        break
                    # convert_output (L160-209)
                    if "<talk>" in text:
                        action = TALK
                    elif re.search(r"\d", text):
                        forward_action = 0
                        goal = self._pixel_goal(text, sim, depth, gps, compass, state.position[1] - initial_height,
                                                to_world)
                        if goal is None:
                            action = STOP
                        else:
                            env.step(LOOKUP)
                            env.step(LOOKUP)
                            if self.append_look_down and look_down_rgb is not None:
                                pol.set_prev_look(e, look_down_rgb)
                            if follower_action(follower.get_next_action(goal)) == STOP:
                                goal, action = None, LEFT
                                pol.clear_conversation(e)
                    else:
                        action_seq = P.parse_actions(text)
                if action is None:
                    if len(action_seq) != 0:
                        action = action_seq.pop(0)
                    elif goal is not None:
                        action = follower_action(follower.get_next_action(goal))
                        forward_action += 1
                        if forward_action > MAX_STEPS or action == STOP:
                            goal, action = None, NOOP
                            pol.clear_conversation(e)
                            if forward_action > MAX_STEPS:
                                forward_action = 0
                    else:
                        action = STOP
                if action != NOOP:
                    last_action = action
                actions.append(action)
                # the evaluator's side (L176-209)
                if action in (STOP, FORWARD, LEFT, RIGHT):
                    obs, _, _, _ = env.step(action)
                    cur = self._own(obs)
                    step_id += 1
                    pol.clear_conversation(e)
                elif action == LOOKDOWN:
                    env.step(action)
                    obs, _, _, _ = env.step(action)
                    cur = self._own(obs)
                elif action == TALK:
                    if len(pol.episodes[e].dialogs) / 2 >= self.turn:
                        npc_answer = QUESTION_LIMIT
                    elif self.npc is None:
                        error = RuntimeError("the agent asked the oracle, and the evaluator has no npc")
                        break
                    else:
                        npc_answer = yield _Request("npc", obs=obs, question=text.replace("<talk>", ""))
                    if npc_answer is None:
                        npc_answer = NO_ANSWER
                elif action != NOOP:
                    error = ValueError("Invalid action %r!" % (action,))
                    break
            st.results.append(self._result(env, episode, scene_id, episode_id, step_id, instruction, path, actions,
                                           error))

    def _pixel_goal(self, text, sim, depth, gps, compass, height, to_world):
        """A pixel answer -> its navigable world goal, or None for a lone number or a point outside the depth frame
        (L165-186): the depth frame filtered, scaled to metres (`* 1000`, `/ 1000`) and lifted through the camera pose
        of this call, taken to the world frame by the episode-start pose and snapped to the navmesh unless navigable."""
        coord = [int(c) for c in re.findall(r"\d+", text)]
        if len(coord) < 2:
            return None
        pixel = [coord[1], coord[0]]
        d = self.depth_filter(depth.reshape(depth.shape[:2]), blur_type=None)
        d = d * (self.max_depth - self.min_depth) + self.min_depth
        d = d * 1000
        x, y = gps
        tf = camera_to_episodic(np.array([x, -y, self.camera_height + height]), compass[0])
        try:
            g = pixel_to_gps(pixel, d / 1000, self.intrinsic, tf)
        except IndexError:
            return None
        goal = (to_world @ np.array([-g[1], 0, -g[0], 1]))[:3]
        if not sim.pathfinder.is_navigable(np.array(goal)):
            goal = np.array(sim.pathfinder.snap_point(np.array(goal)))
        return goal

    def _result(self, env, episode, scene_id, episode_id, step_id, instruction, path, actions, error):
        """The episode's progress.json dict (L218-230), plus the error that ended it, if any."""
        m = env.get_metrics()
        result = {"scene_id": scene_id, "episode_id": episode_id, "success": m["success"], "spl": m["spl"],
                  "os": m["oracle_success"], "ne": m["distance_to_goal"], "steps": step_id,
                  "episode_instruction": instruction, "path": path, "action": actions,
                  "object_category": episode.object_category if "vln" not in self.task else ""}
        if error is not None:
            result["error"], result["error_message"] = type(error).__name__, str(error)
        return result

    @staticmethod
    def _own(obs):
        """Copies of an observation's RGB, depth, gps and compass (a simulator may render into one buffer)."""
        return np.array(obs["rgb"]), np.array(obs["depth"]), np.array(obs["gps"]), np.array(obs["compass"])
