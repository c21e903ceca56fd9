"""System-1 input preprocessing on the GPU (SURVEY.md §8 row a12).

The reference prepares every System-1 call on the host, frame by frame, with Pillow
(internnav/agent/internvla_n1_agent.py L308-334):

    rgb   : np.array(Image.fromarray(rgb).resize((224, 224))) / 255.0
    depth : np.array(Image.fromarray(depth[:, :, 0]).resize((224, 224))) * 10.0, values above 5.0 set to 5.0

for the remembered goal frame and the current frame.  `FramePreprocessor` does the same for all environments of a step
in a handful of launches: raw uint8 / float32 frames are copied to the device once and resampled there by
`n1_resize_rgb_u8` / `n1_resize_f32`, which reproduce Pillow's resampler bit for bit (csrc/resize.cu).  There is no
host fallback: without the library or an H100 the constructor raises.
"""
import ctypes
from ctypes import c_void_p

import numpy as np
import torch

from . import _lib
from ._lib import check

SYS1_DEPTH_THRESHOLD = 5.0
_bound = False


def _bind(L):
    global _bound
    if _bound:
        return
    vp, ci = c_void_p, ctypes.c_int
    L.n1_resize_plan_create.restype = ci
    L.n1_resize_plan_create.argtypes = [ci, ci, ci, ci, ctypes.POINTER(vp), vp]
    L.n1_resize_plan_destroy.restype = None
    L.n1_resize_plan_destroy.argtypes = [vp]
    L.n1_resize_workspace_bytes.restype = ctypes.c_size_t
    L.n1_resize_workspace_bytes.argtypes = [vp, ci, ci]
    L.n1_resize_rgb_u8.restype = ci
    L.n1_resize_rgb_u8.argtypes = [vp, vp, ci, vp, vp, vp, ctypes.c_size_t, vp]
    L.n1_resize_f32.restype = ci
    L.n1_resize_f32.argtypes = [vp, vp, ci, ctypes.c_float, ctypes.c_float, vp, vp, ctypes.c_size_t, vp]
    L.n1_resize_coeffs.restype = ci
    L.n1_resize_coeffs.argtypes = [ci, ci, ci, ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_double),
                                   ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_int32)]
    _bound = True


RESIZE_SYMBOLS = ["n1_resize_plan_create", "n1_resize_plan_destroy", "n1_resize_workspace_bytes", "n1_resize_rgb_u8",
                  "n1_resize_f32", "n1_resize_coeffs"]


def resize_coeffs(in_size, out_size):
    """Host-only: Pillow's per-axis tables as computed by the library -> (bounds [out,2], weights [out,k], fixed [out,k])."""
    L = _lib.lib()
    _bind(L)
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


class FramePreprocessor:
    def __init__(self, device="cuda:0", out_size=224):
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("n1b200 has no CPU path: FramePreprocessor needs device='cuda:N'")
        self.out = out_size
        self._plans, self._ws = {}, {}
        _bind(_lib.lib())

    def __del__(self):
        try:
            L = _lib.lib()
            for p in self._plans.values():
                L.n1_resize_plan_destroy(p)
        except Exception:
            pass

    def _plan(self, h, w):
        p = self._plans.get((h, w))
        if p is None:
            p = c_void_p()
            with torch.cuda.device(self.device):
                check(_lib.lib().n1_resize_plan_create(h, w, self.out, self.out, ctypes.byref(p), _lib.stream_ptr()))
            self._plans[(h, w)] = p
        return p

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
