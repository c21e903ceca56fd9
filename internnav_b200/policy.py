"""Batched dual-system policy: the host side of System 2 (prompt building, image history, answer parsing) and of
System 1 (trajectory -> action ids) for B environments, on top of the n1b200 model mirror.

Mirrors `InternVLAN1Net` (internnav/model/basemodel/internvla_n1/internvla_n1_policy.py): `init_prompts` L60-86,
`reset` L88-94, `parse_actions` L96-102, `step_no_infer` L104-108, `s2_step` L110-198, `s1_step_latent` L200-215 --
per-environment state kept in a list, and the three model calls of one `s2_step` (vision tower + `generate`, then vision
tower + prefill again inside `generate_latents`) replaced by ONE `generate_with_latents` call for the whole batch.

The HF processor (chat template + tokenizer + Qwen2-VL image processor) is injected: it is the reference's own
collaborator (`AutoProcessor.from_pretrained(model_path)`, L44-47) and needs the checkpoint directory, which is not
available offline.  Anything with `apply_chat_template`, `__call__(text=[...], images=[...], return_tensors="pt")` and
`.tokenizer.decode` works (tests use oracle/policy_script.FakeProcessor).

Images take one of two paths.  When the policy runs on a CUDA device and the processor's `image_processor` is one that
`QwenImagePreprocessor` reproduces (the PIL-backed Qwen2-VL processor), every frame is prepared on the device: the
history keeps device uint8 frames, the frames of one call are uploaded and resized together, and the pixel rows of all
environments come from one `QwenImagePreprocessor` call, bit-equal to the processor's.  The processor then only
tokenises the chat text, with each image placeholder expanded as it would expand it.  Otherwise every frame is a PIL
image and the processor prepares each environment's prompt on the host, as in the reference.

A model without a System 1 (`system1 = None`, the System-2-only checkpoint) is served as the reference evaluator serves it
in its `system2` mode: `s2_step` calls `generate` alone (no TRAJ pass), pixel answers carry no latent plan
(`output_latent` is None), and `s1_step_latent` raises.  `system2_only=True` serves any model that way, one with a System
1 included: the evaluator's `system2` mode loads the checkpoint as plain Qwen2.5-VL, so no latent plan is ever computed.
"""
import copy
import itertools
import math
import re
from collections import OrderedDict
from types import SimpleNamespace

import numpy as np
import torch
from PIL import Image

from .postprocess import batched_traj_to_actions, chunk_token, s1_action_list
from .preprocess import QwenImagePreprocessor

DEFAULT_IMAGE_TOKEN = "<image>"
PROMPT = ("You are an autonomous navigation assistant. Your task is to <instruction>. Where should you go next to stay "
          "on track? Please output the next waypoint\'s coordinates in the image. Please output STOP when you have "
          "successfully completed the task.")
CONJUNCTION = "you can see "
ACTIONS2IDX = OrderedDict({"STOP": [0], "↑": [1], "←": [2], "→": [3], "↓": [5]})
_ACTION_RE = re.compile("|".join(re.escape(a) for a in ACTIONS2IDX))


def parse_actions(output):
    """L96-102: every STOP / arrow occurrence, in order, as action ids."""
    return list(itertools.chain.from_iterable(ACTIONS2IDX[m] for m in _ACTION_RE.findall(output)))


def split_and_clean(text):
    """vln_utils.py L19-33: split on <image>, drop newlines and surrounding blanks, skip empty pieces."""
    out = []
    for part in re.split(r"(<image>)", text):
        if part == DEFAULT_IMAGE_TOKEN:
            out.append(part)
        else:
            part = part.replace("\n", "").strip()
            if part:
                out.append(part)
    return out


def _image_tokens(h, w):
    """Merged rows (= image tokens) of an h x w frame, rounded up: at least what the processor's grid gives."""
    return math.ceil(h / 28) * math.ceil(w / 28)


class S2Output(SimpleNamespace):
    def __init__(self):
        super().__init__(output_action=None, output_pixel=None, output_latent=None)


class _Episode:
    """Per-environment conversation state (the instance attributes of the reference class, L52-57 / L88-94).  The frames
    of rgb_list / input_images are PIL images on the host path and device uint8 [H, W, 3] tensors on the device path."""

    def __init__(self):
        self.rgb_list = []
        self.episode_idx = 0
        self.conversation_history = []
        self.llm_output = ""
        self.input_images = []


class InternVLAN1Policy:
    def __init__(self, model, processor, num_envs=1, num_history=8, resize_w=384, resize_h=384, continuous_traj=True,
                 max_new_tokens=128, device=None, vision_cache_frames=0, system2_only=False, kv_pool_tokens=None):
        self.model, self.processor = model, processor
        self.num_history, self.resize_w, self.resize_h = num_history, resize_w, resize_h
        self.continuous_traj = continuous_traj
        self.max_new_tokens = max_new_tokens
        self.device = device if device is not None else getattr(model, "device", "cpu")
        self.has_system1 = getattr(model, "has_system1", True)
        # whether s2_step computes latent plans (generate_with_latents) or calls generate alone
        self.latent_plans = self.has_system1 and not system2_only
        self.episodes = [_Episode() for _ in range(num_envs)]
        # K/V cache of each environment's last System-2 conversation, passed back only on a turn that continues that
        # conversation: here the look-down turn (reference internvla_n1_agent_realworld.py L176 / L226 / L239)
        self._kv_pool = None
        self._kv = [None] * num_envs
        # None: one slot of _kv_capacity tokens per environment.  An integer: a paged pool of that many tokens shared by
        # all environments (each still bounded by _kv_capacity), which evicts the least recently used conversations
        # when it runs out of pages
        self.kv_pool_tokens = None if kv_pool_tokens is None else int(kv_pool_tokens)
        # vision features of images seen in earlier System-2 calls, kept for `vision_cache_frames` resized frames per
        # environment (0: no pool, every call encodes all its images)
        if vision_cache_frames > 0 and getattr(model, "make_feature_pool", None) is None:
            raise ValueError("vision_cache_frames > 0 needs a model with make_feature_pool")
        self.vision_cache_frames = int(vision_cache_frames)
        self._feature_pool = None
        # System-2 images on the device when the processor's image arithmetic can be reproduced there
        self._vl = None
        if torch.device(self.device).type == "cuda":
            self._vl = QwenImagePreprocessor.from_hf(getattr(processor, "image_processor", None), self.device)

    def eval(self):
        return self

    def reset(self, env_ids=None):
        for e in (range(len(self.episodes)) if env_ids is None else env_ids):
            self.episodes[e] = _Episode()
            self._kv[e] = None
            if self._kv_pool is not None and self._kv_pool.paged:
                self._kv_pool.release(e)

    def _kv_capacity(self, frame_h, frame_w):
        """Tokens one environment's slot must hold: a fresh turn (num_history + 1 resized frames), the look-down frame at
        full size, two answers, the TRAJ rows, and 512 tokens for the text of both turns.  A conversation that still
        does not fit runs uncached."""
        nq = getattr(getattr(self.model, "config", None), "n_query", 4)
        return ((self.num_history + 1) * _image_tokens(self.resize_h, self.resize_w) + _image_tokens(frame_h, frame_w) +
                2 * self.max_new_tokens + nq + 512)

    def _feature_rows(self, frame_h, frame_w):
        """Rows of the vision-feature pool: vision_cache_frames resized frames per environment, plus the most one call
        can need at once (every environment's fresh-turn images and its look-down frame)."""
        n, frame = len(self.episodes), _image_tokens(self.resize_h, self.resize_w)
        return n * self.vision_cache_frames * frame + n * ((self.num_history + 1) * frame + _image_tokens(frame_h, frame_w))

    def _features(self, frame_shape):
        """feature_pool for one call, or None without a vision cache."""
        if self.vision_cache_frames <= 0:
            return None
        if self._feature_pool is None:
            self._feature_pool = self.model.make_feature_pool(self._feature_rows(*frame_shape))
        return self._feature_pool

    def _frame_shape(self, rgbs):
        """(height, width) of the raw frames, which size the pools when they are first made."""
        return np.asarray(next(r for r in rgbs if r is not None)).shape[:2]

    def _caches(self, env_ids, continues, frame_shape):
        """past_key_values for one call, or None when the model keeps no K/V caches.  An environment whose turn
        continues its last conversation (continues[i]) gets that conversation's cache back; every other one starts an
        empty cache on its own slot."""
        paged = self.kv_pool_tokens is not None
        make = getattr(self.model, "make_paged_kv_pool" if paged else "make_kv_pool", None)
        if make is None:
            return None
        if self._kv_pool is None:
            self._kv_pool = make(len(self.episodes), self.kv_pool_tokens, self._kv_capacity(*frame_shape)) if paged else \
                make(len(self.episodes), self._kv_capacity(*frame_shape))
        return [self._kv[e] if c and self._kv[e] is not None else self._kv_pool.handle(e)
                for e, c in zip(env_ids, continues)]

    def step_no_infer(self, env_ids, rgbs, depths=None, poses=None):
        if self._vl is not None:
            frames = self._device_frames(rgbs, [True] * len(rgbs))
        else:
            frames = [Image.fromarray(rgb).convert("RGB").resize((self.resize_w, self.resize_h)) for rgb in rgbs]
        for e, frame in zip(env_ids, frames):
            ep = self.episodes[e]
            ep.rgb_list.append(frame)
            ep.episode_idx += 1

    def _device_frames(self, rgbs, resize):
        """Raw frames -> device uint8 frames: each uploaded once, those with resize[i] set resized to resize_h x resize_w
        (Pillow's bicubic), the others kept at full size.  One upload and at most one resize per (shape, resize).  A
        None entry (a turn that brings no new frame) stays None."""
        groups = {}
        for i, rgb in enumerate(rgbs):
            if rgb is None:
                continue
            a = np.asarray(rgb)
            if a.dtype != np.uint8 or a.ndim != 3 or a.shape[-1] != 3:
                a = np.asarray(Image.fromarray(rgb).convert("RGB"))
            groups.setdefault((a.shape, bool(resize[i])), []).append((i, a))
        out = [None] * len(rgbs)
        for (_, rs), members in groups.items():
            x = torch.from_numpy(np.stack([a for _, a in members])).to(self.device)
            if rs:
                x = self._vl.resize(x, (self.resize_h, self.resize_w))
            # every frame owns its memory, so dropping one environment's history frees it
            for k, (i, _) in enumerate(members):
                out[i] = x[k].clone() if len(members) > 1 else x[0]
        return out

    # ------------------------------------------------------------------ System 2
    def _build_inputs(self, ep, rgb, instruction, look_down, conjunction=CONJUNCTION):
        """L113-164 for one environment -> processor output (input_ids [1, S], pixel_values, image_grid_thw)."""
        image = None if rgb is None else Image.fromarray(rgb).convert("RGB")
        if image is not None and not look_down:
            image = image.resize((self.resize_w, self.resize_h))
        chat = self._chat(ep, image, instruction, look_down, conjunction)
        return self.processor(text=[chat], images=ep.input_images, return_tensors="pt")

    def _chat(self, ep, image, instruction, look_down, conjunction=CONJUNCTION):
        """L113-163 for one environment: records the (resized, unless look_down) frame and extends the conversation ->
        the chat text, one image placeholder per image of ep.input_images.  `conjunction` opens the sentence that shows
        the current frame."""
        if not look_down:
            ep.rgb_list.append(image)
            ep.conversation_history = []
            text = PROMPT.replace("<instruction>.", instruction)
            if ep.episode_idx == 0:
                history_id = []
            else:
                history_id = np.unique(np.linspace(0, ep.episode_idx - 1, self.num_history, dtype=np.int32)).tolist()
                text += " These are your historical observations: %s." % ((DEFAULT_IMAGE_TOKEN + "\n") * len(history_id))
            ep.input_images = [ep.rgb_list[i] for i in sorted(history_id)] + ep.rgb_list[-1:]
            img_id = 0
            ep.episode_idx += 1
        else:  # the look-down frame continues the conversation and never enters the history
            ep.input_images.append(image)
            img_id = -1
            assert ep.llm_output != "", "Last llm_output should not be empty when look down"
            text = ""
            ep.conversation_history.append({"role": "assistant", "content": [{"type": "text", "text": ep.llm_output}]})
        text += " %s." % (conjunction + DEFAULT_IMAGE_TOKEN)
        content = []
        for part in split_and_clean(copy.deepcopy(text)):
            if part == DEFAULT_IMAGE_TOKEN:
                content.append({"type": "image", "image": ep.input_images[img_id]})
                img_id += 1
            else:
                content.append({"type": "text", "text": part})
        ep.conversation_history.append({"role": "user", "content": content})
        return self.processor.apply_chat_template(ep.conversation_history, tokenize=False, add_generation_prompt=True)

    def _expand_image_tokens(self, chat, grids):
        """Qwen2_5_VLProcessor.__call__'s text expansion: the k-th image placeholder becomes gh * gw / merge^2 of them."""
        tok = self.processor.image_token
        parts = chat.split(tok)
        assert len(parts) == len(grids) + 1, "%d image placeholders for %d images" % (len(parts) - 1, len(grids))
        merge2 = QwenImagePreprocessor.MERGE ** 2
        return parts[0] + "".join(tok * (int(t * h * w) // merge2) + p for (t, h, w), p in zip(grids.tolist(), parts[1:]))

    def _prepare_device(self, env_ids, rgbs, instructions, look_downs, conjunctions, results):
        """The device path of s2_step's input preparation -> (prepared [(j, input_ids list)], device bf16 pixel rows,
        image_grid_thw); per-environment failures go to results[j]."""
        frames = self._device_frames(rgbs, [not ld for ld in look_downs])
        chats = []
        for j, (e, ins, ld, cj) in enumerate(zip(env_ids, instructions, look_downs, conjunctions)):
            try:
                chats.append((j, self._chat(self.episodes[e], frames[j], ins, ld, cj)))
            except Exception as exc:  # noqa: BLE001 -- reported per environment; the agent applies the retry rule
                results[j] = exc
        if not chats:
            return [], None, None
        pixels, grids = self._vl([im for j, _ in chats for im in self.episodes[env_ids[j]].input_images])
        prepared, g = [], 0
        for j, chat in chats:
            n = len(self.episodes[env_ids[j]].input_images)
            text = self._expand_image_tokens(chat, grids[g:g + n])
            prepared.append((j, self.processor(text=[text], return_tensors="pt")["input_ids"][0].tolist()))
            g += n
        return prepared, pixels, grids

    def s2_step(self, env_ids, rgbs, depths, poses, instructions, intrinsic, look_downs, conjunctions=None):
        """One System-2 consultation for the listed environments (one model call).  Returns a list with, per
        environment, an S2Output (discrete `output_action` list, or `output_pixel` + `output_latent` [1, n_query, H];
        None without a System 1 or with system2_only) or the Exception that environment's host-side preparation raised.  `conjunctions`:
        per environment, the phrase before the current frame's placeholder (default "you can see ", as this policy's
        reference does; the VLN-CE evaluator draws one at random per call)."""
        results = [None] * len(env_ids)
        conjunctions = [CONJUNCTION] * len(env_ids) if conjunctions is None else list(conjunctions)
        if self._vl is not None:
            prepared, pixels, grids = self._prepare_device(env_ids, rgbs, instructions, look_downs, conjunctions, results)
            if not prepared:
                return results
            prompts = [ids for _, ids in prepared]
        else:
            prepared = []
            for j, (e, rgb, ins, ld, cj) in enumerate(zip(env_ids, rgbs, instructions, look_downs, conjunctions)):
                try:
                    prepared.append((j, self._build_inputs(self.episodes[e], rgb, ins, ld, cj)))
                except Exception as exc:  # noqa: BLE001 -- reported per environment; the agent applies the retry rule
                    results[j] = exc
            if not prepared:
                return results
            prompts = [inp["input_ids"][0].tolist() for _, inp in prepared]
            pixels = torch.cat([inp["pixel_values"] for _, inp in prepared], dim=0)
            grids = torch.cat([torch.stack(list(inp["image_grid_thw"])).reshape(-1, 3) for _, inp in prepared], dim=0)
        shape = self._frame_shape([rgbs[j] for j, _ in prepared])
        caches = self._caches([env_ids[j] for j, _ in prepared], [look_downs[j] for j, _ in prepared], shape)
        kw = {} if caches is None else {"past_key_values": caches}
        features = self._features(shape)
        if features is not None:
            kw["feature_pool"] = features
        with torch.no_grad():
            if self.latent_plans:
                out = self.model.generate_with_latents(prompts, pixels, grids, max_new_tokens=self.max_new_tokens, **kw)
            else:
                out = self.model.generate(prompts, pixels, grids, max_new_tokens=self.max_new_tokens,
                                          return_dict_in_generate=True, **kw)
        for n, (j, _) in enumerate(prepared):
            if caches is not None:
                self._kv[env_ids[j]] = out.past_key_values[n]
            ep = self.episodes[env_ids[j]]
            ep.llm_output = self.processor.tokenizer.decode(out.generated[n], skip_special_tokens=True)
            results[j] = self._answer(ep, out, n)
        return results

    def _answer(self, ep, out, n):
        """The S2Output of prompt n of a generate output `out` whose decoded answer is ep.llm_output, or the Exception
        its parsing raised."""
        res = S2Output()
        try:
            if re.search(r"\d", ep.llm_output):   # pixel goal "y x" -> [x, y] plus the latent plan (L179-190)
                coord = [int(c) for c in re.findall(r"\d+", ep.llm_output)]
                res.output_pixel = np.array([int(coord[1]), int(coord[0])])
                res.output_latent = out.latents[n:n + 1] if self.latent_plans else None
            else:
                res.output_action = parse_actions(ep.llm_output)
            return res
        except Exception as exc:  # noqa: BLE001 -- e.g. an answer with a single number (IndexError at L181 as well)
            return exc

    # ------------------------------------------------------------------ System 1
    def s1_step_latent(self, env_ids, rgbs, depths, latents):
        """L200-215 for the listed environments in one generate_traj call: rgbs / depths are the per-environment
        [1, 2, 224, 224, 3] / [1, 2, 224, 224, 1] stacks of the agent, latents the [1, n_query, H] plans."""
        if not self.has_system1:
            raise RuntimeError("s1_step_latent needs a System 1, and the policy's model has none (system1 = None: a "
                               "System-2-only checkpoint answers with discrete actions or pixel goals only)")
        lat = torch.cat([l.reshape(1, *l.shape[-2:]) for l in latents], dim=0)
        rgb = torch.cat([torch.as_tensor(r).reshape(1, *torch.as_tensor(r).shape[-4:]) for r in rgbs], dim=0)
        dep = torch.cat([torch.as_tensor(d).reshape(1, *torch.as_tensor(d).shape[-4:]) for d in depths], dim=0)
        with torch.no_grad():
            traj = self.model.generate_traj(traj_latents=lat, images_dp=rgb.float(), depths_dp=dep.float())
        B = len(env_ids)
        if self.continuous_traj:
            lists = batched_traj_to_actions(traj, B, max_actions=4)
        else:  # one sampled trajectory per environment, tokens -> ids (vln_utils.py L36-60)
            per = traj.shape[0] // B
            lists = [chunk_token(traj.view(B, per, *traj.shape[1:])[b, np.random.choice(per)]) for b in range(B)]
        return [SimpleNamespace(idx=s1_action_list(a)) for a in lists]
