"""Model-level mirror of the reference InternVLA-N1 dual-system model and its policy wrapper.

`InternVLAN1ForCausalLM` keeps the hot-path API surface of the reference class
(internnav/model/basemodel/internvla_n1/internvla_n1.py L39-441): `generate_latents(input_ids, pixel_values,
image_grid_thw)`, `generate_traj(traj_latents, images_dp, depths_dp, ...)`, attributes `.visual`, `.model.navdp`,
`.config.{system1, n_query}`, `.get_model()`, `.device`.  Both systems execute in libn1b200.so; PyTorch carries the
tensors.  Everything is batched over B independent environments, each treated exactly like the reference's single one.

`generate()` is the greedy decode of System 2 (`model.generate(do_sample=False)`, internvla_n1_policy.py L169-176) on a
KV cache; `generate_with_latents()` additionally extends that cache by the TRAJ tokens, which replaces the reference's
second full prefill in `generate_latents(output_ids, ...)` (policy L187-190).

`forward()` is the training forward of the navdp_async branch on a collated batch (the backward lives in train_step.py).

`system1 = "nextdit_async"` (the released DualVLN head: trajectory DiT + flow matching, nextdit.py) and the synchronous
`system1 = "nextdit"` head (the same DiT conditioned on the projected latent plan alone) are served through the same
`generate_traj`; their training branch is not built (the training step is the navdp_async one, train_step.py).

`system1 = None` (no `system1` in config.json: the released System-2 checkpoint) builds System 2 alone, as the reference
class does (internvla_n1_arch.py L121-123): no `latent_queries`, no trajectory head.  `generate()` works as for the dual
model; every call that needs a System 1 raises.  The class is also exported as `Qwen2_5_VLForConditionalGeneration`, the
name under which the reference evaluator loads that checkpoint in its `system2` mode (habitat_vln_evaluator.py L123-129).
"""
from types import SimpleNamespace

import torch

from .navdp import NavDP_Policy_DPT_CriticSum_DAT
from .postprocess import batched_traj_to_actions, s1_action_list
from .qwen import EOS_TOKEN_IDS, PAD_TOKEN_ID, QWEN25VL_7B, System2

TRAJ_TOKEN_INDEX = 151667
IMAGE_TOKEN_INDEX = 151655
# the System-1 configurations built from config.system1 (internvla_n1_arch.py L121-145); None: System 2 only
SYSTEM1_TYPES = (None, "navdp_async", "nextdit_async", "nextdit")
# System-1 modules hanging directly off `.model` (internvla_n1_arch.py L131-145); the RGB branch belongs to nextdit_async
_NEXTDIT_HEADS = ("cond_projector.", "action_encoder.", "action_decoder.", "traj_dit.")
_NEXTDIT_ASYNC_HEADS = _NEXTDIT_HEADS + ("rgb_model.", "memory_encoder.", "rgb_resampler.")


class _Model:
    """Stands in for `InternVLAN1Model` (= `.model` / `.get_model()` of the reference class)."""

    def __init__(self, navdp, s2, config, nextdit=None):
        self.navdp = navdp          # system1 = "navdp_async"
        self.nextdit = nextdit      # system1 = "nextdit_async" / "nextdit": traj_dit, cond_projector, ... in one object
        self._s2 = s2
        self.config = config
        self.device = s2.device

    @property
    def latent_queries(self):
        raise AttributeError("latent_queries live inside the n1b200 handle; pass them through load_state_dict")


class InternVLAN1ForCausalLM:
    def __init__(self, cfg=None, device="cuda:0", system1="navdp_async", predict_size=32, memory_size=2):
        if system1 == "navdp":
            raise NotImplementedError("system1 = 'navdp' (a synchronous NavDP head) is not a configuration the reference "
                                      "builds: its model creates no navdp module for it, so generate_traj cannot run. "
                                      "Use 'navdp_async', 'nextdit_async', 'nextdit' or no system1 (System 2 only)")
        if system1 not in SYSTEM1_TYPES:
            raise NotImplementedError("n1b200 implements system1 = 'navdp_async', 'nextdit_async', 'nextdit' and None "
                                      "(System 2 only); got %r" % (system1,))
        self.cfg = dict(QWEN25VL_7B if cfg is None else cfg)
        self.device = torch.device(device)
        self.config = SimpleNamespace(system1=system1, n_query=self.cfg["n_query"], use_cache=True,
                                      hidden_size=self.cfg["hidden"], image_token_id=IMAGE_TOKEN_INDEX)
        self._s2 = System2(self.cfg, device=device)
        navdp = nextdit = None
        if system1 == "navdp_async":
            navdp = NavDP_Policy_DPT_CriticSum_DAT(memory_size=memory_size, predict_size=predict_size,
                                                   vlm_token_dim=self.cfg["hidden"], navdp_version=0.1, device=device,
                                                   n_query=self.cfg["n_query"])
        elif system1 is not None:
            from .nextdit import NextDiTSystem1
            nextdit = NextDiTSystem1(device=device, asynchronous=system1 == "nextdit_async")
        self.model = _Model(navdp, self._s2, self.config, nextdit)

    @classmethod
    def from_pretrained(cls, model_path, torch_dtype=None, attn_implementation=None, device_map=None, device=None, **kw):
        """`InternVLAN1ForCausalLM.from_pretrained(model_path, torch_dtype=torch.bfloat16, attn_implementation=
        "flash_attention_2", device_map={"": device})` (internvla_n1_policy.py L33-38): reads config.json and the weight
        shards of a checkpoint directory and packs them into the library.  `torch_dtype` / `attn_implementation` are
        accepted for signature compatibility (the kernels are bf16 with fp32 accumulation; attention is the library's).
        The System 1 is config.json's `system1`; without that key the model is System 2 alone, as in the reference."""
        from .checkpoint import read_checkpoint
        if device is None:
            device = (device_map or {}).get("", "cuda:0") if isinstance(device_map, dict) else (device_map or "cuda:0")
        cfg, conf, sd = read_checkpoint(model_path)
        model = cls(cfg, device=str(device), system1=conf.get("system1"),
                    predict_size=int(conf.get("predict_step_nums", 32)))
        model.load_state_dict(sd)
        model.name_or_path = model_path
        return model

    # ------------------------------------------------------------------ reference-shaped accessors
    def get_model(self):
        return self.model

    def get_n_query(self):
        return self.config.n_query

    def get_system1_type(self):
        return self.config.system1

    @property
    def has_system1(self):
        return self.config.system1 is not None

    def _require_system1(self, call):
        if not self.has_system1:
            raise RuntimeError("%s needs a System 1, and this model has none: its config.json names no `system1` (a "
                               "System-2-only checkpoint without latent_queries or a trajectory head); use generate()"
                               % call)

    def eval(self):
        return self

    def visual(self, pixel_values, grid_thw):
        grid = grid_thw.tolist() if torch.is_tensor(grid_thw) else grid_thw
        return self._s2.visual(pixel_values, grid)

    def load_state_dict(self, state_dict, strict=True):
        """Full-model state_dict in the reference checkpoint layout: `visual.*`, `model.*` (incl. `model.latent_queries`
        and `model.navdp.*`; a System-2-only checkpoint has neither).  `lm_head.weight` goes to System 2 (generate())."""
        navdp_sd = {k[len("model.navdp."):]: v for k, v in state_dict.items() if k.startswith("model.navdp.")}
        rest = {k: v for k, v in state_dict.items() if not k.startswith("model.navdp.")}
        if self.model.nextdit is not None:
            # the NextDiT modules hang directly off `.model` in the reference (internvla_n1_arch.py L131-145)
            heads = _NEXTDIT_ASYNC_HEADS if self.model.nextdit.asynchronous else _NEXTDIT_HEADS
            dit_sd = {k[len("model."):]: v for k, v in rest.items() if k.startswith("model.") and k[len("model."):].startswith(heads)}
            rest = {k: v for k, v in rest.items() if not (k.startswith("model.") and k[len("model."):].startswith(heads))}
            self.model.nextdit.load_state_dict(dit_sd)
        self._s2.load_state_dict(rest)
        if navdp_sd:
            self.model.navdp.load_state_dict(navdp_sd)

    def load_parts(self, s2_state_dict, system1_state_dict):
        if not self.has_system1 and system1_state_dict:
            raise ValueError("load_parts: this model has no System 1 to load system1_state_dict into")
        self._s2.load_state_dict(s2_state_dict)
        if self.has_system1:
            (self.model.navdp if self.model.nextdit is None else self.model.nextdit).load_state_dict(system1_state_dict)

    # ------------------------------------------------------------------ hot path
    @staticmethod
    def _prompts(input_ids):
        if torch.is_tensor(input_ids):
            return [row.tolist() for row in input_ids]
        return [list(map(int, p)) for p in input_ids]

    def generate_latents(self, input_ids, pixel_values, image_grid_thw):
        """internvla_n1.py L320-347.  input_ids: [B, S] tensor (equal lengths) or a list of B token-id lists (ragged);
        pixel_values [sum patches, 1176]; image_grid_thw [n_img, 3] in prompt order -> [B, n_query, hidden]."""
        self._require_system1("generate_latents")
        grid = image_grid_thw.tolist() if torch.is_tensor(image_grid_thw) else image_grid_thw
        with torch.no_grad():
            return self._s2.generate_latents(self._prompts(input_ids), pixel_values, grid)

    def generate_traj(self, traj_latents, images_dp, depths_dp=None, predict_step_nums=32, guidance_scale=1.0,
                      num_inference_steps=10, num_sample_trajs=32, x_init=None, step_noise=None):
        """internvla_n1.py L349-441: the nextdit branch (L359-432, flow-matching Euler over the trajectory DiT with
        classifier-free guidance) or the navdp branch (L434-441) -> [num_sample_trajs * B, predict_size, 3]."""
        self._require_system1("generate_traj")
        if self.model.nextdit is not None:
            return self.model.nextdit.generate_traj(traj_latents.to(self.device), images_dp, depths_dp,
                                                    predict_step_nums=predict_step_nums, guidance_scale=guidance_scale,
                                                    num_inference_steps=num_inference_steps,
                                                    num_sample_trajs=num_sample_trajs, x_init=x_init)
        return self.model.navdp.predict_pointgoal_action_async(
            traj_latents.to(self.device), images_dp, depths_dp, sample_num=num_sample_trajs, x_init=x_init,
            step_noise=step_noise)

    def dual_system_step(self, input_ids, pixel_values, image_grid_thw, images_dp, depths_dp, x_init=None,
                         step_noise=None):
        """One full policy step for B environments: System-2 latent plan -> System-1 trajectories -> action ids.
        Returns (trajectories [32B, T, 3], list of B action lists (<= 4 non-zero ids each, [] => action -1))."""
        self._require_system1("dual_system_step")
        lat = self.generate_latents(input_ids, pixel_values, image_grid_thw)
        traj = self.generate_traj(lat, images_dp, depths_dp, x_init=x_init, step_noise=step_noise)
        acts = [s1_action_list(a) for a in batched_traj_to_actions(traj, lat.shape[0], max_actions=4)]
        return traj, acts

    def s1_training_loss(self, traj_hidden_states, traj_images, traj_depths, traj_poses, video_frame_num, noise=None,
                         timesteps=None):
        """The navdp_async branch of the training forward, from the gathered latent states on (internvla_n1.py
        L231-303): traj_hidden_states [B, n_query, H] (the 4 states at t_s_pos); traj_images [B, f, 224, 224, 3];
        traj_depths [B, f, 224, 224]; traj_poses [B, f, 32, 3]; video_frame_num [B] -> scalar loss (the forward; the backward lives in train_step.py)."""
        B, f = traj_images.shape[:2]
        hs = traj_hidden_states.unsqueeze(1).repeat(1, f, 1, 1).flatten(0, 1)
        loss_mask = torch.arange(f, device=traj_images.device).expand(B, f) < video_frame_num.to(traj_images.device).unsqueeze(1)
        cur_images, cur_depths = traj_images.flatten(0, 1), traj_depths.flatten(0, 1)
        goal_images = traj_images[:, 0:1].repeat(1, f, 1, 1, 1).flatten(0, 1)
        goal_depths = traj_depths[:, 0:1].repeat(1, f, 1, 1).flatten(0, 1)
        images_dp = torch.stack([goal_images, cur_images], dim=1)
        depths_dp = torch.stack([goal_depths, cur_depths], dim=1).unsqueeze(-1)
        pred, eps = self.model.navdp.forward_vlm_traj(hs, images_dp, depths_dp, traj_poses, noise=noise,
                                                      timesteps=timesteps)
        err = (pred.float() - eps.float()).square()
        mask = loss_mask.flatten(0, 1)[:, None, None].to(err.device)
        return (err * mask).sum() / mask.sum() / (err.shape[1] * err.shape[2])

    def generate(self, input_ids=None, pixel_values=None, image_grid_thw=None, max_new_tokens=128, do_sample=False,
                 eos_token_id=None, pad_token_id=None, return_dict_in_generate=False, with_latents=False, feature_pool=None,
                 **hf_kwargs):
        """`model.generate(**inputs, max_new_tokens=128, do_sample=False, use_cache=True, past_key_values=None,
        return_dict_in_generate=True).sequences` (internvla_n1_policy.py L169-176) for B prompts.  `sequences` is
        [B, S_max + longest generation] int64: prompt, generated ids (the eos id included), then `pad_token_id`; ragged
        prompts are right-aligned the way the HF processor pads them (left padding).  Other HF keyword arguments
        (attention_mask, use_cache, ...) are accepted and have no effect on greedy search.  `past_key_values`: one KVCache
        (or None) per prompt, from `make_kv_pool(...).handle(slot)` or a previous call's `out.past_key_values`; the
        longest reusable prefix of each prompt is then neither re-encoded nor re-prefilled (qwen.System2.generate),
        and the output also carries `past_key_values` (one new KVCache per prompt), `prefill_rows` and `vit_patches`.
        A None entry next to KVCaches starts a fresh conversation on an unused slot of their pool; a list of None only
        (no pool to write to) is an uncached call.  `feature_pool` (from `make_feature_pool`): the vision tower runs only
        on the images the pool does not hold yet, and the output also carries `image_hits` (images served from the pool)
        and `vit_patches`; outputs are byte-identical to a call without it."""
        if do_sample or hf_kwargs.get("num_beams", 1) != 1:
            raise NotImplementedError("n1b200 implements greedy search only (the reference calls do_sample=False)")
        if with_latents:
            self._require_system1("generate(with_latents=True)")
        eos = EOS_TOKEN_IDS if eos_token_id is None else \
            (tuple(eos_token_id) if isinstance(eos_token_id, (list, tuple)) else (int(eos_token_id),))
        pad = PAD_TOKEN_ID if pad_token_id is None else int(pad_token_id)
        prompts = self._prompts(input_ids)
        grid = image_grid_thw.tolist() if torch.is_tensor(image_grid_thw) else image_grid_thw
        caches = hf_kwargs.get("past_key_values")
        if caches is not None and all(c is None for c in caches):
            caches = None
        extra = {} if caches is None else {"past_key_values": caches}
        if feature_pool is not None:
            extra["feature_pool"] = feature_pool
        with torch.no_grad():
            toks, lat, passes = self._s2.generate(prompts, pixel_values, grid, max_new_tokens=int(max_new_tokens),
                                                  eos_token_ids=eos, pad_token_id=pad, with_latents=with_latents, **extra)
        s_max = max(len(p) for p in prompts)
        g_max = max(len(t) for t in toks)
        seq = torch.full((len(prompts), s_max + g_max), pad, dtype=torch.int64)
        for b, (p, t) in enumerate(zip(prompts, toks)):
            seq[b, s_max - len(p):s_max] = torch.tensor(p, dtype=torch.int64)
            seq[b, s_max:s_max + len(t)] = torch.tensor(t, dtype=torch.int64)
        out = SimpleNamespace(sequences=seq.to(self.device), generated=toks, latents=lat, decode_passes=passes)
        if caches is not None:  # one KVCache per prompt (None: the conversation did not fit its slot)
            info = self._s2.last_cache
            out.past_key_values, out.prefill_rows, out.vit_patches = info["caches"], info["prefill_rows"], info["vit_patches"]
        if feature_pool is not None:
            out.image_hits, out.vit_patches = self._s2.last_features["image_hits"], self._s2.last_features["vit_patches"]
        return out if (return_dict_in_generate or with_latents) else out.sequences

    def make_kv_pool(self, slots, capacity):
        """A K/V cache pool for `slots` conversations of up to `capacity` tokens (prompt + generated + n_query rows),
        allocated once: 2 * layers * kv_heads * head_dim * 2 bytes per token and slot."""
        from .qwen import KVPool
        return KVPool(self._s2, slots, capacity)

    def make_paged_kv_pool(self, slots, tokens, max_tokens_per_slot=None):
        """A paged K/V cache pool: ceil(tokens / 64) pages of 64 tokens shared by `slots` conversations of up to
        `max_tokens_per_slot` tokens each (default: the whole pool).  A conversation holds pages for the tokens it has;
        generate() evicts the least recently used conversations outside a call when the call needs more pages."""
        return self._s2.make_paged_kv_pool(slots, tokens, max_tokens_per_slot)

    def make_feature_pool(self, rows):
        """A vision-feature pool of `rows` merged rows (v_out bf16 each, 7 168 B at the 7B shapes), allocated once; pass it
        as `feature_pool=` to reuse the vision tower's output for images seen in earlier calls."""
        from .qwen import ImageFeaturePool
        return ImageFeaturePool(self._s2, rows)

    def generate_with_latents(self, input_ids, pixel_values, image_grid_thw, max_new_tokens=128, **kw):
        """One System-2 call of the dual-system policy (internvla_n1_policy.py L166-195): greedy answer tokens AND the
        latent plan `generate_latents(output_ids, pixel_values, image_grid_thw)`, sharing one vision pass, one prefill
        and the decode's K/V cache.  -> namespace(sequences, generated, latents [B, n_query, hidden], decode_passes)."""
        self._require_system1("generate_with_latents")
        return self.generate(input_ids, pixel_values, image_grid_thw, max_new_tokens=max_new_tokens, with_latents=True,
                             return_dict_in_generate=True, **kw)

    def traj_hidden_states(self, input_ids, attention_mask, pixel_values, image_grid_thw, t_s_pos):
        """System-2 half of the training forward (internvla_n1.py L128-235) for a collated batch
        (internvla_n1_lerobot_dataset.py L1155-1277: every sample ends with n_query TRAJ tokens at t_s_pos[b], then
        padding; attention_mask = input_ids != pad).  Causal attention makes the states at the TRAJ positions a function
        of the unmasked tokens before them only, and masked tokens are invisible as keys and skipped by get_rope_index,
        so this is the latent-plan prefill over the unmasked prefix of each sample.  -> [B, n_query, hidden]"""
        rows = self._prompts(input_ids)
        nq = self.config.n_query
        mask = None if attention_mask is None else \
            (attention_mask.tolist() if torch.is_tensor(attention_mask) else attention_mask)
        prompts = []
        for b, row in enumerate(rows):
            t = int(t_s_pos[b])
            if row[t:t + nq] != [TRAJ_TOKEN_INDEX] * nq:
                raise ValueError("sample %d: input_ids[t_s_pos : t_s_pos + n_query] are not the TRAJ tokens" % b)
            keep = [True] * len(row) if mask is None else [bool(v) for v in mask[b]]
            if any(tok == IMAGE_TOKEN_INDEX and keep[i] for i, tok in enumerate(row) if i >= t + nq):
                raise NotImplementedError("image tokens after the TRAJ tokens (not produced by the reference collator)")
            prompts.append([tok for i, tok in enumerate(row[:t]) if keep[i]])
        return self.generate_latents(prompts, pixel_values, image_grid_thw)

    def forward(self, input_ids=None, attention_mask=None, labels=None, t_s_pos=None, pixel_values=None,
                image_grid_thw=None, traj_images=None, traj_depths=None, video_frame_num=None, traj_poses=None,
                noise=None, timesteps=None, **hf_kwargs):
        """Training forward of the navdp_async branch (internvla_n1.py L58-318) on a collated batch -> namespace(loss,
        logits=None, traj_hidden_states).  This call is the forward (loss value, no autograd graph); the optimisation step --
        backward kernels, gradient exchange, AdamW -- is `train_step.DualSystemTrainer.step` (SURVEY.md §8 row a13); `logits` (computed but unused by this branch in the reference, L229) are not produced.
        `noise` / `timesteps` inject the draws of `sample_noise` (navdp.py L165-175) for parity tests."""
        self._require_system1("forward")
        if labels is None or t_s_pos is None or traj_images is None:
            raise NotImplementedError("forward() implements the training branch (labels + t_s_pos + traj_* given); for "
                                      "inference use generate() / generate_latents() / generate_traj()")
        hs = self.traj_hidden_states(input_ids, attention_mask, pixel_values, image_grid_thw, t_s_pos)
        loss = self.s1_training_loss(hs, traj_images, traj_depths, traj_poses, video_frame_num, noise=noise,
                                     timesteps=timesteps)
        return SimpleNamespace(loss=loss, logits=None, traj_hidden_states=hs)

    __call__ = forward


Qwen2_5_VLForConditionalGeneration = InternVLAN1ForCausalLM
