"""System-2 image preprocessing on the GPU: QwenImagePreprocessor's rows and grids are bit-equal to the Qwen2-VL image
processor's (converted to bf16, as the model consumes them) for a batch of mixed sizes, its resizes equal Pillow's,
and the policy's device path drives the model exactly as the host path does over a scripted episode."""
import os
import sys

import numpy as np
import pytest
import torch
from PIL import Image

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from vl_processor import qwen_processor  # noqa: E402

pytestmark = pytest.mark.gpu


def _raw(shape, seed):
    return np.random.default_rng(seed).integers(0, 256, (*shape, 3), dtype=np.uint8)


def test_rows_and_grids_equal_the_processor():
    from internnav_b200.preprocess import QwenImagePreprocessor
    ip = qwen_processor(max_pixels=400_000).image_processor
    vl = QwenImagePreprocessor.from_hf(ip, "cuda:0")
    assert isinstance(vl, QwenImagePreprocessor) and (vl.min_pixels, vl.max_pixels) == (3136, 400_000)
    # 384^2 -> 392^2, 480 x 640 -> 476 x 644, width only (392 x 500 -> 392 x 504), identity, raised to min_pixels,
    # clamped to max_pixels, odd sizes; repeated shapes share one resize
    shapes = [(384, 384), (480, 640), (392, 500), (392, 392), (20, 30), (900, 1200), (101, 57), (384, 384), (33, 777)]
    raws = [_raw(s, i) for i, s in enumerate(shapes)]
    px, grids = vl([torch.from_numpy(r).cuda() for r in raws])
    ref = ip(images=[Image.fromarray(r) for r in raws], return_tensors="pt")
    assert torch.equal(grids, ref["image_grid_thw"]), (grids, ref["image_grid_thw"])
    assert grids[5, 1] * grids[5, 2] * 196 <= 400_000 and grids[4, 1] * grids[4, 2] * 196 >= 3136
    assert px.dtype == torch.bfloat16 and px.is_cuda
    assert torch.equal(px.cpu().view(torch.int16), ref["pixel_values"].to(torch.bfloat16).view(torch.int16))


def test_resize_equals_pillow():
    from internnav_b200.preprocess import QwenImagePreprocessor
    vl = QwenImagePreprocessor.from_hf(qwen_processor().image_processor, "cuda:0")
    for (h, w), (oh, ow) in [((480, 640), (384, 384)), ((384, 384), (392, 392)), ((392, 500), (392, 504)),
                             ((392, 392), (392, 392)), ((480, 640), (476, 644)), ((31, 45), (90, 100))]:
        raws = np.stack([_raw((h, w), 10 + k) for k in range(3)])
        got = vl.resize(raws, (oh, ow))               # host input
        assert got.is_cuda and got.shape == (3, oh, ow, 3)
        assert torch.equal(vl.resize(torch.from_numpy(raws).cuda(), (oh, ow)), got)   # device input
        for k in range(3):
            want = np.asarray(Image.fromarray(raws[k]).resize((ow, oh)))
            assert np.array_equal(got[k].cpu().numpy(), want), ((h, w), (oh, ow), k)


class _HostOnly:
    """The processor without its image_processor attribute: the policy takes the host path."""

    def __init__(self, p):
        self._p, self.tokenizer = p, p.tokenizer

    def apply_chat_template(self, *a, **k):
        return self._p.apply_chat_template(*a, **k)

    def __call__(self, *a, **k):
        return self._p(*a, **k)


class _Recorder:
    """Forwards the model; records each generate_with_latents call's prompts, pixel-row bytes, ids and latents."""

    def __init__(self, model):
        self.m, self.config, self.device, self.calls = model, model.config, model.device, []

    def make_kv_pool(self, slots, capacity):
        return self.m.make_kv_pool(slots, capacity)

    def generate_with_latents(self, prompts, pixels, grids, **kw):
        lens = [len(c) for c in kw["past_key_values"]]   # before the call makes the handles stale
        out = self.m.generate_with_latents(prompts, pixels, grids, **kw)
        self.calls.append(dict(prompts=prompts, rows=pixels.to(torch.bfloat16).cpu().view(torch.int16),
                               grids=torch.as_tensor(grids).cpu(), reused=lens, generated=out.generated,
                               latents=out.latents.cpu(), prefill=out.prefill_rows))
        return out


def test_policy_device_path_matches_host_path():
    from internnav_b200.internvla_n1 import InternVLAN1ForCausalLM
    from internnav_b200.manifest import random_navdp_state_dict
    from internnav_b200.policy import InternVLAN1Policy
    from oracle import qwen_oracle as Q
    cfg = Q.tiny_cfg()
    model = InternVLAN1ForCausalLM(cfg, device="cuda:0")
    model.load_parts(Q.make_s2_state_dict(cfg, seed=5, lm_head=True), random_navdp_state_dict(seed=6, vlm_token_dim=cfg["hidden"]))
    proc = qwen_processor()
    dev, host = _Recorder(model), _Recorder(model)
    kw = dict(num_envs=3, num_history=4, resize_w=100, resize_h=90, max_new_tokens=6)
    pd, ph = InternVLAN1Policy(dev, proc, **kw), InternVLAN1Policy(host, _HostOnly(proc), **kw)
    assert pd._vl is not None and ph._vl is None

    def frame(k, e, shape=(96, 128)):
        return _raw(shape, 100 * k + e)

    def s2(env_ids, k, look_downs):
        outs = []
        for pol in (pd, ph):
            res = pol.s2_step(env_ids, [frame(k, e, (120, 90) if e == 2 else (96, 128)) for e in env_ids], None, None,
                              ["go to door %d" % e for e in env_ids], None, look_downs)
            assert all(not isinstance(r, Exception) for r in res), res
            outs.append(res)
        return outs

    for k in range(3):   # environment 2 sees frames of another shape
        for pol in (pd, ph):
            pol.step_no_infer([0, 1, 2], [frame(k, e, (120, 90) if e == 2 else (96, 128)) for e in range(3)])
    assert all(f.is_cuda and f.shape == (90, 100, 3) for f in pd.episodes[0].rgb_list)
    assert all(np.array_equal(f.cpu().numpy(), np.asarray(g)) for f, g in zip(pd.episodes[2].rgb_list, ph.episodes[2].rgb_list))
    s2([0, 1, 2], 3, [False] * 3)             # fresh turns with history
    s2([0, 2], 4, [True, True])               # look-down turns continue on the K/V pool
    s2([1, 0], 5, [True, False])              # a look-down and a fresh turn in one call
    assert len(dev.calls) == len(host.calls) == 3
    for a, b in zip(dev.calls, host.calls):
        assert a["prompts"] == b["prompts"]
        assert torch.equal(a["grids"], b["grids"]) and torch.equal(a["rows"], b["rows"])
        assert a["reused"] == b["reused"] and a["generated"] == b["generated"] and a["prefill"] == b["prefill"]
        assert torch.equal(a["latents"], b["latents"])
    assert dev.calls[1]["reused"][0] > 0 and dev.calls[1]["prefill"] < sum(len(p) for p in dev.calls[1]["prompts"])

    # reset drops the environment's device frames
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    n_frames = len(pd.episodes[1].rgb_list) + 1   # history + the look-down frame
    assert n_frames >= 5
    pd.reset([1])
    assert pd.episodes[1].rgb_list == [] and pd.episodes[1].input_images == []
    freed = before - torch.cuda.memory_allocated()
    assert freed >= (n_frames - 1) * 90 * 100 * 3 + 96 * 128 * 3, freed
