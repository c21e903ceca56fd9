"""The batched VL-LN dialog evaluator and the text-only continuation it relies on, on the GPU: the reference traces
(tests/golden/habitat_dialog_traces.json) with the policy on the device; a closed loop on the library's kernels (tiny
Qwen2.5-VL config, seeded weights) whose answers include questions to a scripted oracle; and `System2.generate` on
batches whose prompts bring no new image."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import habitat_dialog_script as D
from oracle import habitat_s2_script as S
from oracle import habitat_script as H

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
with open(os.path.join(ROOT, "tests", "golden", "habitat_dialog_traces.json"), encoding="utf-8") as fh:
    TRACES = json.load(fh)["traces"]


@pytest.mark.parametrize("ti", range(len(TRACES)))
def test_device_policy_reproduces_trace(ti):
    ev = D.replay([TRACES[ti]], device="cuda:0")
    assert ev.policy.device == torch.device("cuda:0")


def test_device_policy_side_by_side_with_one_buffer_environments():
    traces = [t for t in TRACES if t["case"]["task"] == "instance_dialog"]
    ev = D.replay(traces, device="cuda:0", reuse_buffer=True)
    assert ev.calls["s2"] <= ev.calls["rounds"]


# ------------------------------------------------------------------------------------------------ closed loop
SMALL_H, SMALL_W = 96, 128


class _Processor:
    """Stand-in for the HF processor with real shapes: characters -> token ids, every image -> a [1, 8, 8] patch grid
    whose pixel rows are seeded by the image's bytes.  `decode` turns the random model's generated ids into a question
    ("<talk>"), a pixel answer inside the 128 x 96 frame, look-down, arrows or STOP, chosen by the ids and by the
    conversation's length: neither a question nor a look-down takes a step, so a conversation that already holds
    MAX_TURNS answers gets arrows instead, and every episode ends.  The processor is called once per prompt, in the
    order the answers are decoded, and queues each conversation's answer count for `decode`."""
    MAX_TURNS = 3

    class _Tok:
        padding_side = "left"

        def __init__(self):
            self.turns = []

        def decode(self, ids, skip_special_tokens=True):
            ids = [int(i) for i in ids if int(i) < 151643] or [0]
            kind = ids[0] % 8
            if self.turns.pop(0) >= _Processor.MAX_TURNS and kind in (0, 1, 4):
                kind = 6
            if kind < 2:
                return "<talk>is it near room %d?" % (ids[-1] % 9)
            if kind < 4:
                return "%d, %d" % ((ids[0] * 7) % SMALL_W, ids[-1] % SMALL_H)
            if kind == 4:
                return "↓"
            if kind == 5 and ids[-1] % 4 == 0:
                return "STOP"
            return "".join("↑←→"[i % 3] for i in ids[:3])

    def __init__(self):
        self.tokenizer = self._Tok()

    def apply_chat_template(self, conversation, tokenize=False, add_generation_prompt=True):
        return "\n".join(t["role"] + ":" + "".join("<image>" if c["type"] == "image" else c["text"] for c in t["content"])
                         for t in conversation)

    def __call__(self, text, images, return_tensors="pt"):
        self.tokenizer.turns.append(text[0].count("\nassistant:"))
        ids, rows, grids = [], [], []
        pieces = text[0].split("<image>")
        for i, piece in enumerate(pieces):
            ids += [1000 + (ord(c) % 5000) for c in piece[-48:]]
            if i < len(pieces) - 1:
                seed = int(np.asarray(images[i], dtype=np.int64).sum()) % (2 ** 31)
                rows.append(torch.randn(64, 1176, generator=torch.Generator().manual_seed(seed)))
                grids.append(torch.tensor([1, 8, 8]))
                ids += [151652] + [151655] * 16 + [151653]
        return {"input_ids": torch.tensor([ids]), "pixel_values": torch.cat(rows), "image_grid_thw": torch.stack(grids)}


class _Env(D.DialogEnv):
    """DialogEnv with 96 x 128 frames (cut from the 480 x 640 ones)."""

    def _observe(self):
        obs = super()._observe()
        return dict(obs, rgb=np.ascontiguousarray(obs["rgb"][::5, ::5]), depth=np.ascontiguousarray(obs["depth"][::5, ::5]))


class _NoPool:
    """The model without `make_kv_pool`: every call re-prefills its whole prompt."""

    def __init__(self, model):
        self.m = model
        self.device, self.config = model.device, model.config
        self.has_system1 = getattr(model, "has_system1", False)

    def generate(self, *a, **kw):
        return self.m.generate(*a, **kw)

    def make_feature_pool(self, rows):
        return self.m.make_feature_pool(rows)


@pytest.fixture(scope="module")
def s2_model():
    from internnav_b200.internvla_n1 import InternVLAN1ForCausalLM
    from oracle import qwen_oracle as Q
    cfg = Q.tiny_cfg()
    m = InternVLAN1ForCausalLM(cfg, device="cuda:0", system1=None)
    m.load_parts(Q.make_s2_state_dict(cfg, seed=3, lm_head=True), None)
    return m


def _npc(questions):
    return [None if len(q) % 5 == 0 else "it is %d rooms to the %s" % (len(q) % 4, "left" if len(q) % 2 else "right")
            for e, env, obs, q in questions]


def _closed_loop(model, robots, vision_cache_frames=0, record=None, capacity=None):
    """Run robots' environments (2 instance-dialog episodes each, 10 steps at most) in one evaluator -> (per robot:
    results and env log, the evaluator).  `record`: list that gets (turn kinds, prompt lengths, generate output, reused
    rows) per System-2 call.  `capacity`: the K/V slot size in tokens."""
    from internnav_b200 import habitat_dialog as HD
    ev = HD.HabitatDialogEvaluator(model, _Processor(), task="instance_dialog", turn=2, num_history=4, resize_w=112,
                                   resize_h=112, max_steps_per_episode=10, max_new_tokens=6, depth_filter=H.depth_filter,
                                   npc=_npc, seeds=[40 + r for r in robots], camera_height=S.CAMERA_HEIGHT,
                                   width=SMALL_W, height=SMALL_H, hfov=S.HFOV, vision_cache_frames=vision_cache_frames,
                                   make_follower=lambda env: D.Follower(env._env.sim, 0.25, False))
    logs = {r: [] for r in robots}
    envs = [_Env(r, 50 + r, 2, logs[r]) for r in robots]
    if record is not None or capacity is not None:
        ev.policy = HD.DialogPolicy(model, ev.processor, num_envs=len(robots), num_history=4, resize_w=112, resize_h=112,
                                    max_new_tokens=6, device=ev.device, vision_cache_frames=vision_cache_frames,
                                    prompt=ev.prompt, turn=2, frame_shape=(SMALL_H, SMALL_W))
        if capacity is not None:
            ev.policy._kv_capacity = lambda h, w: capacity
        if record is not None:
            generate, s2_step = model.generate, ev.policy.s2_step
            kinds = []

            def step(env_ids, rgbs, depths, poses, turns, *a, **kw):
                kinds[:] = [t.kind for t in turns]
                return s2_step(env_ids, rgbs, depths, poses, turns, *a, **kw)

            def gen(prompts, *a, **kw):
                out = generate(prompts, *a, **kw)
                record.append((list(kinds), [len(p) for p in prompts], out, list(model._s2.last_cache["reused"])))
                return out
            ev.policy.s2_step, model.generate = step, gen
    try:
        res = ev.run(envs)
    finally:
        if record is not None:
            del model.generate
    return [(rs, logs[r]) for r, rs in zip(robots, res)], ev


def test_closed_loop_batched_equals_single_environment_drivers(s2_model):
    robots = [0, 1, 2, 3]
    batched, ev = _closed_loop(s2_model, robots)
    again, _ = _closed_loop(s2_model, robots)
    assert batched == again, "two runs differ"
    for j, r in enumerate(robots):
        single, _ = _closed_loop(s2_model, [r])
        assert single[0] == batched[j], "robot %d differs from its single-environment driver" % r
    print("calls", ev.calls, "results", [b[0] for b in batched])
    assert ev.calls["s2"] >= 2 and ev.calls["s2"] <= ev.calls["rounds"]
    assert ev.calls["npc"] >= 1      # the loop asked the oracle
    assert all(len(b[0]) == 2 for b in batched)


def test_closed_loop_with_and_without_pools_is_byte_identical(s2_model):
    robots = [0, 1, 2]
    want, _ = _closed_loop(_NoPool(s2_model), robots)
    assert _closed_loop(s2_model, robots)[0] == want
    assert _closed_loop(s2_model, robots, vision_cache_frames=4)[0] == want
    assert _closed_loop(_NoPool(s2_model), robots, vision_cache_frames=4)[0] == want


def test_dialog_turns_prefill_only_their_text(s2_model):
    """Every dialog turn continues its conversation's K/V slot (it prefills fewer rows than its prompt holds), a call of
    dialog turns only runs no vision tower, and a conversation beyond its slot's capacity runs uncached with the same
    answers."""
    record = []
    got, _ = _closed_loop(s2_model, [0, 1, 2, 3], record=record)
    dialog = [(n, r) for kinds, lens, out, reused in record for k, n, r in zip(kinds, lens, reused) if k == "dialog"]
    assert dialog, "no dialog turn"
    assert all(0 < r < n for n, r in dialog), dialog
    for kinds, lens, out, reused in record:
        if all(k == "dialog" for k in kinds):
            assert out.vit_patches == 0 and out.prefill_rows == sum(n - r for n, r in zip(lens, reused))
    print("dialog turns", len(dialog), "calls", len(record),
          "dialog-only calls", sum(all(k == "dialog" for k in rec[0]) for rec in record))
    small, _ = _closed_loop(s2_model, [0, 1, 2, 3], capacity=120)   # most conversations overflow their slot
    assert small == got


# ------------------------------------------------------------------------------------------------ System2.generate
def _setup(seed):
    from internnav_b200.qwen import System2
    from oracle import qwen_oracle as Q
    cfg = Q.tiny_cfg()
    s2 = System2(cfg, device="cuda:0")
    s2.load_state_dict(Q.make_s2_state_dict(cfg, seed=seed, lm_head=True))
    return s2


def _px(grids, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(sum(t * h * w for t, h, w in grids), 1176, generator=g).bfloat16().cuda()


@pytest.mark.parametrize("features", [False, True])
def test_text_only_continuations_in_mixed_and_image_free_batches(features):
    """One batch of a dialog continuation (text only), a look-down continuation and a fresh prompt, then a batch of
    dialog continuations only (no new image: no features, no vision tower, a row table of 0 rows): every prompt's
    tokens equal the prompt run alone and uncached."""
    from internnav_b200.qwen import ImageFeaturePool, KVPool
    from oracle import qwen_oracle as Q
    s2 = _setup(41)
    rng = np.random.Generator(np.random.PCG64(41))
    fp = ImageFeaturePool(s2, 512) if features else None
    kw = {} if fp is None else {"feature_pool": fp}
    gA, gB, gC, gl = [(1, 8, 8), (1, 8, 12)], [(1, 8, 8)], [(1, 12, 8)], (1, 12, 16)
    pA, pB, pC = Q.make_prompt(rng, 10, gA, 6), Q.make_prompt(rng, 7, gB, 5), Q.make_prompt(rng, 8, gC, 3)
    pxA, pxB, pxC, pxl = _px(gA, 1), _px(gB, 2), _px(gC, 3), _px([gl], 4)
    pool = KVPool(s2, 4, 1024)
    t1, _, _ = s2.generate([pA, pB, pC], torch.cat([pxA, pxB, pxC]), gA + gB + gC, max_new_tokens=5,
                           past_key_values=[pool.handle(0), pool.handle(1), pool.handle(2)], **kw)
    hA, hB, hC = s2.last_cache["caches"]

    def alone(p, px, grids):
        return s2.generate([p], px, grids, max_new_tokens=5)[0][0]

    # dialog (A: answer + text), look-down (B: answer + text + a new image), fresh (D)
    pA2 = pA + t1[0] + Q.make_prompt(rng, 9, [], 0)
    pB2 = pB + t1[1] + Q.make_prompt(rng, 4, [gl], 3)
    gD = [(1, 8, 8)]
    pD = Q.make_prompt(rng, 6, gD, 4)
    pxD = _px(gD, 5)
    nA, nB = len(hA), len(hB)
    toks, _, _ = s2.generate([pA2, pB2, pD], torch.cat([pxA, pxB, pxl, pxD]), gA + gB + [gl] + gD, max_new_tokens=5,
                             past_key_values=[hA, hB, None], **kw)
    info = s2.last_cache
    assert info["reused"] == [nA, nB, 0], info["reused"]
    assert info["vit_patches"] == 12 * 16 + 8 * 8     # the look-down frame and the fresh prompt's image only
    for b, (p, px, grids) in enumerate([(pA2, pxA, gA), (pB2, torch.cat([pxB, pxl]), gB + [gl]), (pD, pxD, gD)]):
        assert toks[b] == alone(p, px, grids), b
    hA2, _, _ = info["caches"]
    nA2, nC = len(hA2), len(hC)
    # dialog continuations only: A again, and C
    pA3 = pA2 + toks[0] + Q.make_prompt(rng, 7, [], 0)
    pC2 = pC + t1[2] + Q.make_prompt(rng, 11, [], 0)
    toks, _, _ = s2.generate([pA3, pC2], torch.cat([pxA, pxC]), gA + gC, max_new_tokens=5, past_key_values=[hA2, hC],
                             **kw)
    info = s2.last_cache
    assert info["vit_patches"] == 0
    assert info["reused"] == [nA2, nC] and info["prefill_rows"] == (len(pA3) - nA2) + (len(pC2) - nC)
    if features:
        assert s2.last_features["vit_patches"] == 0
    for b, (p, px, grids) in enumerate([(pA3, pxA, gA), (pC2, pxC, gC)]):
        assert toks[b] == alone(p, px, grids), b
