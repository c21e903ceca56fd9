"""The policy's look-down turn on the GPU: InternVLAN1Policy keeps each environment's K/V cache, passes it back on that
environment's look-down turn only, and drops it on a fresh turn and on reset.  The model is the tiny Qwen config behind
the public InternVLAN1ForCausalLM.generate_with_latents; the processor is a stand-in whose tokenizer round-trips the
generated ids, as a real chat template does, so the look-down prompt really extends the previous conversation."""
import re

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

_AZ = "abcdefghijklmnopqrstuvwxyz"


def _b26(i):
    return "".join(_AZ[(i // 26 ** k) % 26] for k in range(3, -1, -1))


class LookDownProcessor:
    """Every answer decodes to its ids as "[wxyz]" groups followed by "↓" (the look-down arrow, no digits); the chat
    template and the tokenizer map those groups back to the same ids.  Other characters are one token each; every image
    is a [1, 8, 8] grid (16 tokens) whose pixel rows are seeded by the frame's content."""

    class _Tok:
        def decode(self, ids, skip_special_tokens=True):
            return "".join("[%s]" % _b26(int(i)) for i in ids) + "↓"

    def __init__(self):
        self.tokenizer = self._Tok()

    def apply_chat_template(self, conversation, tokenize=False, add_generation_prompt=True):
        parts = [turn["role"] + ":" + "".join("<image>" if c["type"] == "image" else c["text"] for c in turn["content"])
                 for turn in conversation]
        return "\n".join(parts) + ("\nassistant:" if add_generation_prompt else "")

    def __call__(self, text, images, return_tensors="pt"):
        ids, rows, grids, k = [], [], [], 0
        for m in re.finditer(r"<image>|\[([a-z]{4})\]|.", text[0], flags=re.S):
            if m.group(0) == "<image>":
                g = torch.Generator().manual_seed(int(np.asarray(images[k]).reshape(-1)[0]))
                rows.append(torch.randn(64, 1176, generator=g))
                grids.append(torch.tensor([1, 8, 8]))
                ids += [151652] + [151655] * 16 + [151653]
                k += 1
            elif m.group(1):
                ids.append(sum(_AZ.index(c) * 26 ** (3 - j) for j, c in enumerate(m.group(1))))
            else:
                ids.append(1000 + ord(m.group(0)) % 5000)
        return {"input_ids": torch.tensor([ids]), "pixel_values": torch.cat(rows), "image_grid_thw": torch.stack(grids)}


class _Recorder:
    """Forwards generate_with_latents and records (prompts, reused-length of each cache passed or None, output)."""

    def __init__(self, model):
        self.m, self.config, self.device, self.calls = model, model.config, model.device, []

    def generate_with_latents(self, prompts, pixels, grids, **kw):
        caches = kw.get("past_key_values")
        lens = None if caches is None else [len(c) for c in caches]
        out = self.m.generate_with_latents(prompts, pixels, grids, **kw)
        self.calls.append((prompts, lens, out))
        return out


class _PoolRecorder(_Recorder):
    def make_kv_pool(self, slots, capacity):
        return self.m.make_kv_pool(slots, capacity)


def _frame(k, e):
    return np.full((48, 64, 3), (31 * e + 7 * k + 3) % 256, dtype=np.uint8)


def _s2(pol, env_ids, k, look_downs):
    res = pol.s2_step(env_ids, [_frame(k, e) for e in env_ids], None, None, ["walk to the door %d" % e for e in env_ids],
                      None, look_downs)
    assert all(not isinstance(r, Exception) for r in res), res
    assert all(r.output_action and r.output_action[-1] == 5 for r in res)  # every answer ends in "↓"
    return res


def _rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm()).item()


def test_policy_look_down_turn_prefills_only_the_new_turn():
    from internnav_b200.internvla_n1 import InternVLAN1ForCausalLM
    from internnav_b200.manifest import random_navdp_state_dict
    from internnav_b200.policy import InternVLAN1Policy
    from oracle import qwen_oracle as Q
    cfg = Q.tiny_cfg()
    model = InternVLAN1ForCausalLM(cfg, device="cuda:0")
    model.load_parts(Q.make_s2_state_dict(cfg, seed=5, lm_head=True), random_navdp_state_dict(seed=6, vlm_token_dim=cfg["hidden"]))
    cached, plain = _PoolRecorder(model), _Recorder(model)   # the second model has no make_kv_pool
    pols = [InternVLAN1Policy(m, LookDownProcessor(), num_envs=2, num_history=4, resize_w=112, resize_h=112,
                              max_new_tokens=6) for m in (cached, plain)]
    pc, pp = pols
    for pol in pols:
        for k in range(3):
            pol.step_no_infer([0, 1], [_frame(k, e) for e in (0, 1)])

    # 1. fresh turn, both environments: empty caches in, outputs byte-identical to the model without a pool
    for pol in pols:
        _s2(pol, [0, 1], 3, [False, False])
    (p1, lens, out_c), (p1_plain, lens_plain, out_p) = cached.calls[-1], plain.calls[-1]
    assert lens == [0, 0] and lens_plain is None and p1 == p1_plain
    assert out_c.prefill_rows == sum(len(p) for p in p1)
    assert out_c.generated == out_p.generated and torch.equal(out_c.latents, out_p.latents)
    assert [len(pc._kv[e]) for e in (0, 1)] == [len(p1[e]) + len(out_c.generated[e]) for e in (0, 1)]

    # 2. look-down turn of environment 0: the cache is passed back and only the new turn is prefilled
    for pol in pols:
        _s2(pol, [0], 4, [True])
    (p2, lens, out_c), (p2_plain, _, out_p) = cached.calls[-1], plain.calls[-1]
    assert p2 == p2_plain
    prev = p1[0] + cached.calls[-2][2].generated[0]
    assert lens == [len(prev)] and p2[0][:len(prev)] == prev      # the template re-tokenises the answer exactly
    assert out_c.prefill_rows == len(p2[0]) - len(prev) and out_c.vit_patches == 64
    assert out_c.generated == out_p.generated and _rel(out_c.latents, out_p.latents) < 1e-2
    assert len(pc._kv[0]) == len(p2[0]) + len(out_c.generated[0])

    # 3. fresh turn of environment 0: its cache is not passed back (an empty one is), and it matches the plain model
    for pol in pols:
        _s2(pol, [0], 5, [False])
    (p3, lens, out_c), (_, _, out_p) = cached.calls[-1], plain.calls[-1]
    assert lens == [0] and out_c.prefill_rows == len(p3[0])
    assert out_c.generated == out_p.generated and torch.equal(out_c.latents, out_p.latents)

    # 4. reset drops environment 1's cache; its next fresh turn starts empty and a look-down after it reuses again
    pc.reset([1])
    assert pc._kv[1] is None
    for k in range(2):
        pc.step_no_infer([1], [_frame(10 + k, 1)])
    _s2(pc, [1], 12, [False])
    p4, lens, out4 = cached.calls[-1]
    assert lens == [0] and out4.prefill_rows == len(p4[0])
    _s2(pc, [1], 13, [True])
    p5, lens, out5 = cached.calls[-1]
    assert lens == [len(p4[0]) + len(out4.generated[0])] and out5.prefill_rows == len(p5[0]) - lens[0]
