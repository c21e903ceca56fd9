"""System-2 image preprocessing on the host side (no GPU): the Qwen2-VL arithmetic that QwenImagePreprocessor and
n1_vl_patchify restate -- smart_resize, the rescale + normalise table, the patch-row order -- against the installed
transformers processor; which processors qualify for the device path; the argument checks of n1_vl_patchify; the
text expansion of the policy's device path against the processor's; the by-shape batching of the resize calls; and a
spill-free compile of the kernel."""
import ctypes
import math
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch
from PIL import Image

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from vl_processor import qwen_processor  # noqa: E402

from internnav_b200.preprocess import QwenImagePreprocessor, by_shape, smart_resize  # noqa: E402

pil_qwen = pytest.importorskip("transformers.models.qwen2_vl.image_processing_pil_qwen2_vl")


def _spec_rows(img, lut):
    """The patch-row order n1_vl_patchify writes, restated: row r of an image is merged block r // 4 (row-major over
    gh / 2 x gw / 2), sub-patch (r % 4) // 2, (r % 4) % 2; element e = c * 392 + t * 196 + py * 14 + px is
    lut[c, pixel (py, px) of that patch], the same for t = 0 and 1."""
    h, w, _ = img.shape
    gw = w // 14
    r = np.arange((h // 14) * gw)[:, None]
    e = np.arange(1176)[None, :]
    b, sub = r // 4, r % 4
    y = ((b // (gw // 2)) * 2 + sub // 2) * 14 + (e % 196) // 14
    x = ((b % (gw // 2)) * 2 + sub % 2) * 14 + (e % 196) % 14
    c = e // 392
    return lut[c, img[y, x, c]]


def test_smart_resize_matches_transformers():
    from transformers.models.qwen2_vl.image_processing_qwen2_vl import smart_resize as ref
    sizes = [1, 3, 13, 14, 27, 28, 29, 41, 42, 55, 56, 57, 100, 224, 383, 384, 392, 480, 500, 640, 1000, 2000, 4000]
    for min_p, max_p in ((56 * 56, 28 * 28 * 1280), (3136, 12845056), (200_000, 400_000)):
        for h in sizes:
            for w in sizes:
                try:
                    want = ref(h, w, 28, min_p, max_p)
                except ValueError:
                    with pytest.raises(ValueError, match="aspect ratio"):
                        smart_resize(h, w, 28, min_p, max_p)
                    continue
                assert smart_resize(h, w, 28, min_p, max_p) == want, (h, w, min_p, max_p)
    # the grid covers the clamps and the error
    assert smart_resize(20, 30, 28, 3136, 10 ** 7)[0] * smart_resize(20, 30, 28, 3136, 10 ** 7)[1] >= 3136
    assert math.prod(smart_resize(2000, 4000, 28, 3136, 400_000)) <= 400_000
    with pytest.raises(ValueError):
        smart_resize(1, 201)


def test_lut_matches_rescale_and_normalize():
    ip = pil_qwen.Qwen2VLImageProcessorPil()
    lut = QwenImagePreprocessor.lut(ip)
    img = np.stack([np.roll(np.arange(256, dtype=np.uint8), 17 * c) for c in range(3)])[:, None, :]   # [3, 1, 256]
    want = ip.normalize(ip.rescale(img, 1 / 255), ip.image_mean, ip.image_std)
    assert want.dtype == np.float32
    assert np.array_equal(lut[np.arange(3)[:, None, None], img], want)


@pytest.mark.parametrize("shape", [(56, 56), (384, 384), (480, 640), (392, 500), (392, 392), (20, 30), (101, 57)])
def test_patch_order_matches_processor(shape):
    """Pillow's uint8 bicubic to the smart_resize size, then the table and the row order above, equal the processor's
    float32 rows bit for bit."""
    ip = pil_qwen.Qwen2VLImageProcessorPil()
    rng = np.random.default_rng(shape[0] * 1000 + shape[1])
    raw = rng.integers(0, 256, (*shape, 3), dtype=np.uint8)
    ref = ip(images=[Image.fromarray(raw)], return_tensors="np")
    oh, ow = smart_resize(*shape, 28, *QwenImagePreprocessor.pixel_limits(ip))
    resized = np.asarray(Image.fromarray(raw).resize((ow, oh), Image.Resampling.BICUBIC))
    assert ref["image_grid_thw"].tolist() == [[1, oh // 14, ow // 14]]
    assert np.array_equal(_spec_rows(resized, QwenImagePreprocessor.lut(ip)), ref["pixel_values"])


def test_qualification_rule():
    from transformers.models.qwen2_vl.image_processing_qwen2_vl import Qwen2VLImageProcessor
    ok = pil_qwen.Qwen2VLImageProcessorPil()
    assert QwenImagePreprocessor.supports(ok)
    assert QwenImagePreprocessor.from_hf(ok, "cpu") is None          # the device path needs a CUDA device
    assert QwenImagePreprocessor.pixel_limits(pil_qwen.Qwen2VLImageProcessorPil(min_pixels=1000, max_pixels=9000)) \
        == (1000, 9000)
    refused = [Qwen2VLImageProcessor(),                                      # torchvision-backed: another bicubic
               pil_qwen.Qwen2VLImageProcessorPil(resample=Image.Resampling.BILINEAR),
               pil_qwen.Qwen2VLImageProcessorPil(patch_size=16),
               pil_qwen.Qwen2VLImageProcessorPil(merge_size=4),
               pil_qwen.Qwen2VLImageProcessorPil(temporal_patch_size=1),
               pil_qwen.Qwen2VLImageProcessorPil(do_normalize=False),
               pil_qwen.Qwen2VLImageProcessorPil(do_rescale=False),
               pil_qwen.Qwen2VLImageProcessorPil(do_resize=False),
               pil_qwen.Qwen2VLImageProcessorPil(rescale_factor=1 / 127.5),
               None, object()]
    for ip in refused:
        assert not QwenImagePreprocessor.supports(ip), ip
        assert QwenImagePreprocessor.from_hf(ip, "cuda:0") is None, ip


def test_vl_patchify_argument_errors():
    """Every argument check runs before the device is touched, so the codes are the same with and without a GPU."""
    from internnav_b200 import _lib
    L = _lib.lib()
    fake = ctypes.c_void_p(1 << 20)
    ws = L.n1_vl_patchify_workspace_bytes(2)
    assert ws >= 2 * ctypes.sizeof(_lib.VlImage) and ctypes.sizeof(_lib.VlImage) == 24

    def call(table, n_rows, ws_bytes=ws, lut=fake, out=fake):
        arr = (_lib.VlImage * len(table))(*[_lib.VlImage(*t) for t in table])
        return L.n1_vl_patchify(arr, len(table), lut, out, n_rows, fake, ws_bytes, None), L.n1_last_error().decode()

    good = [(1 << 20, 392, 392, 0), (1 << 21, 476, 644, 784)]
    rows = 784 + 17 * 23
    assert call(good, rows, lut=None)[0] == -2                                 # N1_ERR_ARG
    assert call(good, rows, out=None)[0] == -2
    assert call([(None, 392, 392, 0), good[1]], rows)[0] == -2
    rc, msg = call([good[0], (1 << 21, 476, 650, 784)], rows)
    assert rc == -2 and "multiples of 28" in msg
    rc, msg = call([good[0], (1 << 21, 476, 644, 700)], rows)
    assert rc == -2 and "starts at row" in msg
    rc, msg = call(good, rows + 1)
    assert rc == -2 and "rows" in msg
    rc, msg = call(good, rows, ws_bytes=ws - 1)
    assert rc == -7 and "workspace" in msg                                     # N1_ERR_WORKSPACE
    assert L.n1_vl_patchify(None, 1, fake, fake, 784, fake, ws, None) == -2


def _episode_turns(policy, processor):
    """A fresh turn with 8 history frames + the current one, then its look-down turn: (chat, images) of each."""
    from internnav_b200.policy import _Episode
    rng = np.random.default_rng(5)
    ep = _Episode()
    for _ in range(12):
        ep.rgb_list.append(Image.fromarray(rng.integers(0, 256, (384, 384, 3), dtype=np.uint8)))
    ep.episode_idx = 12
    frame = Image.fromarray(rng.integers(0, 256, (384, 384, 3), dtype=np.uint8))
    fresh = policy._chat(ep, frame, "walk to the kitchen door", False)
    fresh_images = list(ep.input_images)
    ep.llm_output = "abcd qrst"
    down = policy._chat(ep, Image.fromarray(rng.integers(0, 256, (480, 640, 3), dtype=np.uint8)), "", True)
    return [(fresh, fresh_images), (down, list(ep.input_images))]


def test_expanded_text_ids_match_processor():
    """The device path tokenises the chat text with each image placeholder expanded as Qwen2_5_VLProcessor.__call__
    expands it; the ids equal the processor's own for a fresh 9-image turn and the look-down turn after it."""
    from internnav_b200.policy import InternVLAN1Policy
    proc = qwen_processor()
    pol = InternVLAN1Policy(model=None, processor=proc, num_envs=1, device="cpu")
    limits = QwenImagePreprocessor.pixel_limits(proc.image_processor)
    turns = _episode_turns(pol, proc)
    assert [len(im) for _, im in turns] == [9, 10]
    for chat, images in turns:
        grids = torch.tensor([(1, *(s // 14 for s in smart_resize(im.height, im.width, 28, *limits))) for im in images])
        ref = proc(text=[chat], images=images, return_tensors="pt")
        assert torch.equal(grids, ref["image_grid_thw"])
        mine = proc(text=[pol._expand_image_tokens(chat, grids)], return_tensors="pt")["input_ids"]
        assert torch.equal(mine, ref["input_ids"])
    with pytest.raises(AssertionError, match="placeholders"):
        pol._expand_image_tokens(turns[0][0], grids[:3])


def test_by_shape_calls_once_per_shape_and_keeps_input_order():
    frames = [np.full((2, 3), 0), np.full((4, 5), 1), np.full((2, 3), 2), np.full((4, 5), 3), np.full((1, 1), 4)]
    calls = []

    def fn(fs):
        calls.append([int(f.flat[0]) for f in fs])
        return [10 * int(f.flat[0]) for f in fs]
    assert by_shape(frames, fn) == [0, 10, 20, 30, 40]
    assert sorted(calls) == [[0, 2], [1, 3], [4]]
    batch = torch.arange(6).reshape(3, 2)   # one shape: fn's own result, no regrouping
    assert by_shape([np.zeros(2)] * 3, lambda fs: batch) is batch


def test_patchify_kernel_compiles_without_spills(tmp_path):
    from internnav_b200 import build
    if not os.path.exists(build.NVCC):
        pytest.skip("nvcc not installed")
    cmd = [build.NVCC] + build.FLAGS + ["-c", os.path.join(build.CSRC, "vl_patch.cu"), "-o", str(tmp_path / "k.o")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    found = re.findall(r"Function properties for (\S*vl_patchify_kernel\S*)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes "
                       r"spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(found) == 1, r.stderr[-2000:]
    assert tuple(int(v) for v in found[0][1:]) == (0, 0, 0), found
