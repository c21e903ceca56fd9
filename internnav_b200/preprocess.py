"""System-1 and System-2 input preprocessing on the GPU (SURVEY.md §8 rows a12 and 8f).

The reference prepares every System-1 call on the host, frame by frame, with Pillow
(internnav/agent/internvla_n1_agent.py L308-334):

    rgb   : np.array(Image.fromarray(rgb).resize((224, 224))) / 255.0
    depth : np.array(Image.fromarray(depth[:, :, 0]).resize((224, 224))) * 10.0, values above 5.0 set to 5.0

for the remembered goal frame and the current frame.  `FramePreprocessor` does the same for all environments of a step
in a handful of launches: raw uint8 / float32 frames are copied to the device once and resampled there by
`n1_resize_rgb_u8` / `n1_resize_f32`, which reproduce Pillow's resampler bit for bit (csrc/resize.cu).  There is no
host fallback: without the library or an H100 the constructor raises.

The reference prepares every System-2 image on the host as well: the policy resizes each frame with Pillow, and the
Qwen2-VL image processor then resizes every image of the prompt again (to `smart_resize`'s multiple of 28), rescales,
normalises and cuts it into 14 x 14 x 2 patch rows in numpy.  `QwenImagePreprocessor` does the same on the device and
produces the processor's rows bit for bit (converted to bf16, as the model consumes them): both resizes on
`n1_resize_rgb_u8` (uint8 output), and rescale + normalise + patchify in one `n1_vl_patchify` launch, since after a
uint8 resize the processor's arithmetic is a table of the 256 byte values per channel.

`System1Inputs` is the System-1 half of the batched drivers (the real-world agent and the VLN-CE evaluator): the 224 x 224
RGB frames, each environment's goal frames, the [goal, current] stacks and the `generate_traj` call.
"""
import math
import ctypes
from ctypes import c_void_p

import numpy as np
import torch
from PIL import Image

from . import _lib
from ._lib import VlImage, check

S1_SIZE = 224
SYS1_DEPTH_THRESHOLD = 5.0


def by_shape(frames, fn):
    """fn over the frames in one call per distinct frame shape (one in all for a fleet of identical cameras).  fn takes a
    list of frames of one shape and returns one result per frame.  -> the per-frame results in input order: fn's own
    return value when all frames have one shape, else a list."""
    groups = {}
    for k, f in enumerate(frames):
        groups.setdefault(tuple(np.shape(f)), []).append(k)
    if len(groups) == 1:
        return fn(list(frames))
    out = [None] * len(frames)
    for idx in groups.values():
        for k, r in zip(idx, fn([frames[k] for k in idx])):
            out[k] = r
    return out


def resize_coeffs(in_size, out_size):
    """Host-only: Pillow's per-axis tables as computed by the library -> (bounds [out,2], weights [out,k], fixed [out,k])."""
    L = _lib.lib()
    cap = 4 * max(1, -(-in_size // out_size)) + 8
    b = (ctypes.c_int32 * (out_size * 2))()
    w = (ctypes.c_double * (out_size * cap))()
    f = (ctypes.c_int32 * (out_size * cap))()
    k = ctypes.c_int32()
    check(L.n1_resize_coeffs(in_size, out_size, cap, b, w, f, ctypes.byref(k)))
    k = k.value
    return (np.frombuffer(b, dtype=np.int32).reshape(out_size, 2).copy(),
            np.frombuffer(w, dtype=np.float64)[: out_size * k].reshape(out_size, k).copy(),
            np.frombuffer(f, dtype=np.int32)[: out_size * k].reshape(out_size, k).copy())


class _ResizePlans:
    """Resize plans on one device, one per (input, output) shape, created on first use and destroyed with the cache."""

    def __init__(self, device):
        self.device, self._plans = device, {}

    def __del__(self):
        try:
            L = _lib.lib()
            for p in self._plans.values():
                L.n1_resize_plan_destroy(p)
        except Exception:
            pass

    def __call__(self, in_h, in_w, out_h, out_w):
        key = (in_h, in_w, out_h, out_w)
        p = self._plans.get(key)
        if p is None:
            p = c_void_p()
            with torch.cuda.device(self.device):
                check(_lib.lib().n1_resize_plan_create(in_h, in_w, out_h, out_w, ctypes.byref(p), _lib.stream_ptr()))
            self._plans[key] = p
        return p


class FramePreprocessor:
    def __init__(self, device="cuda:0", out_size=S1_SIZE):
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("n1b200 has no CPU path: FramePreprocessor needs device='cuda:N'")
        self.out = out_size
        self._plans, self._ws = _ResizePlans(self.device), {}

    def _plan(self, h, w):
        return self._plans(h, w, self.out, self.out)

    def _scratch(self, key, nbytes):
        k = (key, torch.cuda.current_stream().cuda_stream)
        buf = self._ws.get(k)
        if buf is None or buf.numel() < nbytes:
            buf = torch.empty(int(nbytes) + 256, dtype=torch.uint8, device=self.device)
            self._ws[k] = buf
        return buf

    def rgb(self, frames):
        """frames uint8 [n, H, W, 3] (tensor or array, host or device) -> float32 [n, 224, 224, 3] in [0, 1]."""
        x = torch.as_tensor(frames)
        assert x.dtype == torch.uint8 and x.ndim == 4 and x.shape[-1] == 3, "rgb frames must be uint8 [n, H, W, 3]"
        x = x.to(self.device).contiguous()
        n, h, w = x.shape[:3]
        L, plan = _lib.lib(), self._plan(h, w)
        out = torch.empty(n, self.out, self.out, 3, dtype=torch.float32, device=self.device)
        nb = L.n1_resize_workspace_bytes(plan, n, 0)
        ws = self._scratch("rgb", nb)
        with torch.cuda.device(self.device):
            check(L.n1_resize_rgb_u8(plan, _lib.ptr(x), n, _lib.ptr(out), None, _lib.ptr(ws), nb, _lib.stream_ptr()))
        return out

    def depth(self, frames, mul=10.0, clip_max=SYS1_DEPTH_THRESHOLD):
        """frames float32 [n, H, W] -> float32 [n, 224, 224] = resized * mul with values above clip_max set to it."""
        x = torch.as_tensor(frames)
        assert x.dtype == torch.float32 and x.ndim == 3, "depth frames must be float32 [n, H, W]"
        x = x.to(self.device).contiguous()
        n, h, w = x.shape
        L, plan = _lib.lib(), self._plan(h, w)
        out = torch.empty(n, self.out, self.out, dtype=torch.float32, device=self.device)
        nb = L.n1_resize_workspace_bytes(plan, n, 1)
        ws = self._scratch("depth", nb)
        with torch.cuda.device(self.device):
            check(L.n1_resize_f32(plan, _lib.ptr(x), n, float(mul), float(clip_max), _lib.ptr(out), _lib.ptr(ws), nb,
                                  _lib.stream_ptr()))
        return out

    def s1_frames(self, goal_rgbs, goal_depths, rgbs, depths):
        """Per-environment lists of raw frames (rgb uint8 [H, W, 3], depth float32 [H, W, 1]) -> the System-1 inputs
        of all environments: float32 [B, 2, 224, 224, 3] and [B, 2, 224, 224, 1], [goal frame, current frame]."""
        B = len(rgbs)
        rgb = np.stack([np.asarray(f) for pair in zip(goal_rgbs, rgbs) for f in pair])
        dep = np.stack([np.asarray(f, dtype=np.float32)[:, :, 0] for pair in zip(goal_depths, depths) for f in pair])
        r = self.rgb(torch.from_numpy(rgb)).view(B, 2, self.out, self.out, 3)
        d = self.depth(torch.from_numpy(dep)).view(B, 2, self.out, self.out, 1)
        return r, d


class System1Inputs:
    """System 1 of a batched driver: [goal frame, current frame] of each listed environment -> one `generate_traj` call.

    The current frames are resized to 224 x 224 as the reference's agents resize them with Pillow: on the device by the
    driver's `FramePreprocessor` (bit-equal), without one by Pillow itself.  The frame of a goal step becomes that
    environment's goal frame, already resized (the reference resizes the same bytes again on every step, with the same
    result), until the next goal step or `reset`.  `depth` is the plain resize of the real-world agent; a driver with
    another depth rule (the VLN-CE evaluator) prepares its depth frames itself.  What happens to the trajectories is the
    driver's."""

    def __init__(self, model, preprocessor=None, x_init=None):
        """`preprocessor`: the FramePreprocessor of the driver's CUDA device, or None (Pillow on the host).  `x_init`:
        None (System 1 draws its initial noise on the device) or a callable env_ids -> noise [len(env_ids) * 32, T, 3]
        for those environments, in that order."""
        self.model, self.preprocessor, self.x_init = model, preprocessor, x_init
        self._goal = {}

    def reset(self, env_ids):
        for e in env_ids:
            self._goal.pop(e, None)

    def rgb(self, frames):
        """Raw uint8 frames [H, W, 3] -> float32 [n, 224, 224, 3] = Pillow-resized / 255, on the driver's device."""
        if self.preprocessor is None:
            return torch.from_numpy(np.stack([np.array(Image.fromarray(np.asarray(f)).resize((S1_SIZE, S1_SIZE))) / 255.0
                                              for f in frames])).float()
        return self._stack(by_shape(frames, lambda fs: self.preprocessor.rgb(np.stack(fs))))

    def depth(self, frames):
        """Raw float32 depth [H, W] (or [H, W, 1]) -> float32 [n, 224, 224], Pillow-resized (mode F), no scaling, no
        clip."""
        frames = [np.asarray(f, dtype=np.float32).reshape(np.shape(f)[:2]) for f in frames]
        if self.preprocessor is None:
            return torch.from_numpy(np.stack([np.array(Image.fromarray(f).resize((S1_SIZE, S1_SIZE))) for f in frames]))
        resize = lambda fs: self.preprocessor.depth(np.stack(fs), mul=1.0, clip_max=float("inf"))  # noqa: E731
        return self._stack(by_shape(frames, resize))

    @staticmethod
    def _stack(rows):
        return rows if torch.is_tensor(rows) else torch.stack(rows)

    def generate(self, env_ids, goals, rgb, depth, latents):
        """The listed environments' current frames, prepared by the driver -- rgb [n, 224, 224, 3], depth [n, 224, 224]
        or None for a System 1 that reads no depth -- and latent plans [.., n_query, H] -> the trajectories of one
        `generate_traj` call.  The frames of the environments in `goals` become their goal frames first."""
        for k, e in enumerate(env_ids):
            if e in goals:
                self._goal[e] = (rgb[k].clone(), None if depth is None else depth[k].clone())
        rgb = torch.stack([torch.stack((self._goal[e][0], rgb[k])) for k, e in enumerate(env_ids)])
        if depth is not None:
            depth = torch.stack([torch.stack((self._goal[e][1], depth[k])) for k, e in enumerate(env_ids)])[..., None]
        lat = torch.cat([l.reshape(1, *l.shape[-2:]) for l in latents])
        kw = {} if self.x_init is None else {"x_init": self.x_init(env_ids)}
        with torch.no_grad():
            return self.model.generate_traj(lat, rgb, depth, **kw)


def smart_resize(height, width, factor=28, min_pixels=56 * 56, max_pixels=28 * 28 * 1280):
    """The size the Qwen2-VL image processor resizes an image to (transformers `smart_resize`): both sides rounded to a
    multiple of `factor`; if that holds more than `max_pixels` pixels, both sides are scaled down by the same factor
    and floored to a multiple (at least `factor`), if fewer than `min_pixels`, scaled up and ceiled.  An aspect ratio
    above 200 is an error."""
    if max(height, width) / min(height, width) > 200:
        raise ValueError("absolute aspect ratio must be smaller than 200, got %r" % (max(height, width) / min(height, width)))
    h_bar, w_bar = round(height / factor) * factor, round(width / factor) * factor
    if h_bar * w_bar > max_pixels:
        beta = math.sqrt((height * width) / max_pixels)
        h_bar = max(factor, math.floor(height / beta / factor) * factor)
        w_bar = max(factor, math.floor(width / beta / factor) * factor)
    elif h_bar * w_bar < min_pixels:
        beta = math.sqrt(min_pixels / (height * width))
        h_bar, w_bar = math.ceil(height * beta / factor) * factor, math.ceil(width * beta / factor) * factor
    return h_bar, w_bar


def _is_pil_qwen2vl(image_processor):
    """True for the PIL/numpy-backed Qwen2-VL image processor: Qwen2VLImageProcessorPil in transformers 5, the slow
    Qwen2VLImageProcessor (not a BaseImageProcessorFast) in transformers 4.  The torchvision-backed processor resizes
    with a different bicubic and is not reproduced."""
    try:
        from transformers.models.qwen2_vl import image_processing_qwen2_vl as qv
    except ImportError:
        return False
    try:
        from transformers.models.qwen2_vl.image_processing_pil_qwen2_vl import Qwen2VLImageProcessorPil
    except ImportError:   # transformers 4
        from transformers.image_processing_utils_fast import BaseImageProcessorFast
        return type(image_processor) is qv.Qwen2VLImageProcessor and not isinstance(image_processor, BaseImageProcessorFast)
    return type(image_processor) is Qwen2VLImageProcessorPil


class QwenImagePreprocessor:
    """The Qwen2-VL image processor of the System-2 prompt images on the GPU, bit-equal to its `pixel_values` converted
    to bf16.  Build it with `from_hf`, which declines any processor whose arithmetic it does not reproduce."""

    PATCH, TEMPORAL, MERGE = 14, 2, 2
    ROW = 3 * TEMPORAL * PATCH * PATCH   # 1176

    def __init__(self, device, lut, min_pixels, max_pixels):
        """lut: bf16 [3, 256] = the processor's rescale + normalise of each byte value per channel."""
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("n1b200 has no CPU path: QwenImagePreprocessor needs device='cuda:N'")
        self.min_pixels, self.max_pixels = int(min_pixels), int(max_pixels)
        self.table = lut.to(self.device, torch.bfloat16).contiguous().reshape(3 * 256)
        self._plans = _ResizePlans(self.device)

    @classmethod
    def supports(cls, image_processor):
        """True for the PIL-backed Qwen2-VL image processor with Pillow bicubic resizing, resize + rescale by 1/255 +
        normalise on, and patch 14 / temporal patch 2 / merge 2: the processor whose rows this class reproduces."""
        from PIL import Image
        ip = image_processor
        if not _is_pil_qwen2vl(ip):
            return False
        try:
            bicubic = int(ip.resample) == int(Image.Resampling.BICUBIC)
        except (TypeError, ValueError):
            return False
        return bool(bicubic and ip.do_resize and ip.do_rescale and ip.do_normalize and ip.rescale_factor == 1 / 255) \
            and (ip.patch_size, ip.temporal_patch_size, ip.merge_size) == (cls.PATCH, cls.TEMPORAL, cls.MERGE)

    @staticmethod
    def pixel_limits(image_processor):
        """(min_pixels, max_pixels) of a Qwen2-VL image processor."""
        size = getattr(image_processor, "size", None) or {}
        return (size["shortest_edge"] if "shortest_edge" in size else image_processor.min_pixels,
                size["longest_edge"] if "longest_edge" in size else image_processor.max_pixels)

    @staticmethod
    def lut(image_processor):
        """float32 [3, 256]: the processor's own rescale + normalise of every byte value of each channel."""
        ip = image_processor
        v = np.broadcast_to(np.arange(256, dtype=np.uint8), (3, 1, 256)).copy()   # channels first
        out = ip.normalize(ip.rescale(v, ip.rescale_factor, input_data_format="channels_first"), ip.image_mean,
                           ip.image_std, input_data_format="channels_first")
        return np.ascontiguousarray(out, dtype=np.float32).reshape(3, 256)

    @classmethod
    def from_hf(cls, image_processor, device):
        """An instance for an image processor `supports` accepts on a CUDA device; None for any other processor or
        device.  The table is converted to bf16 as the model converts the processor's float32 rows."""
        if torch.device(device).type != "cuda" or not cls.supports(image_processor):
            return None
        return cls(device, torch.from_numpy(cls.lut(image_processor)).to(torch.bfloat16),
                   *cls.pixel_limits(image_processor))

    def size(self, h, w):
        """(h, w) an image of h x w pixels is resized to."""
        return smart_resize(h, w, self.PATCH * self.MERGE, self.min_pixels, self.max_pixels)

    def grid(self, h, w):
        """image_grid_thw row of an h x w image: (1, gh, gw) patches."""
        oh, ow = self.size(h, w)
        return 1, oh // self.PATCH, ow // self.PATCH

    def resize(self, frames, size):
        """frames uint8 [n, H, W, 3] (tensor or array, host or device) -> device uint8 [n, h, w, 3], Pillow's bicubic
        `Image.resize((w, h))` of each frame."""
        x = torch.as_tensor(frames)
        assert x.dtype == torch.uint8 and x.ndim == 4 and x.shape[-1] == 3, "frames must be uint8 [n, H, W, 3]"
        x = x.to(self.device).contiguous()
        (n, h, w), (oh, ow) = x.shape[:3], size
        L, plan = _lib.lib(), self._plans(h, w, oh, ow)
        out = torch.empty(n, oh, ow, 3, dtype=torch.uint8, device=self.device)
        nb = L.n1_resize_workspace_bytes(plan, n, 0)
        ws = torch.empty(max(nb, 1), dtype=torch.uint8, device=self.device)
        with torch.cuda.device(self.device):
            check(L.n1_resize_rgb_u8(plan, _lib.ptr(x), n, None, _lib.ptr(out), _lib.ptr(ws), nb, _lib.stream_ptr()))
        return out

    def __call__(self, images):
        """images: device uint8 [H, W, 3] frames -> (pixel_values bf16 [N, 1176] on the device, image_grid_thw int64
        [n, 3]), as `processor(images=...)` returns them.  One resize per distinct frame shape, one patchify launch."""
        assert len(images) > 0, "no images"
        for im in images:
            assert im.dtype == torch.uint8 and im.ndim == 3 and im.shape[-1] == 3, "images must be uint8 [H, W, 3]"
        resized = by_shape(images, lambda ims: self.resize(torch.stack(ims), self.size(*ims[0].shape[:2])))
        table = (VlImage * len(images))()
        rows = 0
        for t, r in zip(table, resized):
            t.src_u8, t.h, t.w, t.row0 = r.data_ptr(), r.shape[0], r.shape[1], rows
            rows += (r.shape[0] // self.PATCH) * (r.shape[1] // self.PATCH)
        L = _lib.lib()
        px = torch.empty(rows, self.ROW, dtype=torch.bfloat16, device=self.device)
        nb = L.n1_vl_patchify_workspace_bytes(len(images))
        ws = torch.empty(nb, dtype=torch.uint8, device=self.device)
        with torch.cuda.device(self.device):
            check(L.n1_vl_patchify(table, len(images), _lib.ptr(self.table), _lib.ptr(px), rows, _lib.ptr(ws), nb,
                                   _lib.stream_ptr()))
        grids = torch.tensor([[1, r.shape[0] // self.PATCH, r.shape[1] // self.PATCH] for r in resized], dtype=torch.int64)
        return px, grids
