"""ctypes binding of libn1b200.so (include/n1b200.h).  PyTorch is used for device memory and streams only.

There is deliberately no fallback: if the shared library is missing, or no sm_90 device is present when a
compute entry point is called, the call raises.
"""
import ctypes
import os
import threading

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libn1b200.so")

_lib = None
_lock = threading.Lock()

c_void_p, c_int, c_size_t, c_float, c_char_p = (
    ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t, ctypes.c_float, ctypes.c_char_p)
c_int32, c_int64, c_double = ctypes.c_int32, ctypes.c_int64, ctypes.c_double
i32p = ctypes.POINTER(c_int32)


class N1Error(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("n1b200 error %d: %s" % (code, msg))
        self.code = code


class TensorDesc(ctypes.Structure):
    _fields_ = [("name", c_char_p), ("data", c_void_p), ("dtype", ctypes.c_int32), ("ndim", ctypes.c_int32),
                ("shape", ctypes.c_int64 * 4)]


class S1Dims(ctypes.Structure):
    _fields_ = [("token_dim", ctypes.c_int32), ("heads", ctypes.c_int32), ("layers", ctypes.c_int32),
                ("predict_size", ctypes.c_int32), ("memory_size", ctypes.c_int32),
                ("vlm_token_dim", ctypes.c_int32), ("n_query", ctypes.c_int32)]


class NavdpPolicyDims(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int32) for n in ("token_dim", "heads", "layers", "predict_size", "memory_size", "depth_frames",
                                              "goal_slots", "ddpm_steps")]


class S2Dims(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int32) for n in ("v_depth", "v_hidden", "v_heads", "v_inter", "v_patch", "v_tpatch",
                                              "v_merge", "v_window", "v_out", "n_fullatt")] + \
               [("fullatt", ctypes.c_int32 * 16)] + \
               [(n, ctypes.c_int32) for n in ("layers", "hidden", "heads", "kv_heads", "head_dim", "inter", "vocab")] + \
               [("rms_eps", ctypes.c_float), ("rope_theta", ctypes.c_float), ("mrope", ctypes.c_int32 * 3),
                ("n_query", ctypes.c_int32)]


class VlImage(ctypes.Structure):
    """n1_vl_image: one resized frame of n1_vl_patchify."""
    _fields_ = [("src_u8", c_void_p), ("h", ctypes.c_int32), ("w", ctypes.c_int32), ("row0", ctypes.c_int64)]


# every symbol include/n1b200.h declares: name -> (restype, argtypes)
SYMBOLS = {
    "n1_version": (c_char_p, []),
    "n1_device_ok": (c_int, [c_int]),
    "n1_create": (c_int, [ctypes.POINTER(c_void_p), c_int]),
    "n1_destroy": (None, [c_void_p]),
    "n1_last_error": (c_char_p, []),
    "n1_s1_load": (c_int, [c_void_p, ctypes.POINTER(S1Dims), ctypes.POINTER(TensorDesc), c_int, c_void_p]),
    "n1_workspace_bytes": (c_size_t, [c_void_p, c_int, c_int, c_int, c_int]),
    "n1_rgbd_encode": (c_int, [c_void_p, c_void_p, c_size_t, c_void_p, c_void_p, c_void_p, c_int, c_void_p]),
    "n1_goal_compress": (c_int, [c_void_p, c_void_p, c_size_t, c_void_p, c_void_p, c_int, c_void_p]),
    "n1_navdp_eps": (c_int, [c_void_p, c_void_p, c_size_t, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p,
                             c_int, c_int, c_int, c_void_p]),
    "n1_navdp_sample": (c_int, [c_void_p, c_void_p, c_size_t, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                c_int, c_int, c_int, c_int, c_void_p]),
    "n1_navdp_policy_load": (c_int, [c_void_p, ctypes.POINTER(NavdpPolicyDims), ctypes.POINTER(TensorDesc), c_int,
                                     c_void_p]),
    "n1_navdp_critic": (c_int, [c_void_p, c_void_p, c_size_t, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "n1_ddpm_tables": (c_int, [c_int, ctypes.POINTER(c_float)]),
    # System 2
    "n1_s2_load": (c_int, [c_void_p, ctypes.POINTER(S2Dims), ctypes.POINTER(TensorDesc), c_int, c_void_p]),
    "n1_s2_has_latent_queries": (c_int, [c_void_p]),
    "n1_s2_has_lm_head": (c_int, [c_void_p]),
    "n1_vit_plan_create": (c_int, [c_void_p, i32p, c_int, ctypes.POINTER(c_void_p), c_void_p]),
    "n1_vit_plan_destroy": (None, [c_void_p]),
    "n1_vit_plan_patches": (c_int64, [c_void_p]),
    "n1_llm_plan_create": (c_int, [c_void_p, i32p, i32p, c_int, i32p, c_int, c_int, c_void_p, i32p, i32p,
                                   ctypes.POINTER(c_void_p), c_void_p]),
    "n1_llm_plan_destroy": (None, [c_void_p]),
    "n1_llm_plan_tokens": (c_int64, [c_void_p]),
    "n1_llm_plan_image_tokens": (c_int64, [c_void_p]),
    "n1_llm_plan_positions": (c_int, [c_void_p, i32p, i32p]),
    "n1_vit_workspace_bytes": (c_size_t, [c_void_p, c_void_p]),
    "n1_llm_workspace_bytes": (c_size_t, [c_void_p, c_void_p]),
    "n1_qwen_vit": (c_int, [c_void_p, c_void_p, c_void_p, c_size_t, c_void_p, c_void_p, c_int64, i32p, c_int64, c_void_p]),
    "n1_llm_prefill": (c_int, [c_void_p, c_void_p, c_void_p, c_size_t, c_void_p, c_void_p, c_void_p]),
    "n1_llm_generate": (c_int, [c_void_p, c_void_p, c_void_p, c_size_t, c_void_p, c_int64, i32p, c_int64, i32p, c_int,
                                c_int32, i32p, i32p, c_void_p, i32p, c_void_p]),
    "n1_kv_pool_create": (c_int, [c_void_p, c_int, c_int, ctypes.POINTER(c_void_p)]),
    "n1_kv_pool_destroy": (None, [c_void_p]),
    "n1_kv_pool_bytes": (c_size_t, [c_void_p]),
    "n1_kv_pool_valid": (c_int, [c_void_p, c_int]),
    "n1_kv_pool_read": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "n1_kv_pool_create_paged": (c_int, [c_void_p, c_int, c_int, c_int, ctypes.POINTER(c_void_p)]),
    "n1_kv_pool_release": (c_int, [c_void_p, c_int]),
    "n1_kv_pool_free_pages": (c_int, [c_void_p]),
    "n1_kv_pool_slot_pages": (c_int, [c_void_p, c_int]),
    "n1_kv_pages_create": (c_int, [c_int, c_int, c_int, ctypes.POINTER(c_void_p)]),
    "n1_kv_pages_destroy": (None, [c_void_p]),
    "n1_kv_pages_prepare": (c_int, [c_void_p, c_int, i32p, i32p, i32p, i32p]),
    "n1_kv_pages_trim": (c_int, [c_void_p, c_int, c_int]),
    "n1_kv_pages_table": (c_int, [c_void_p, i32p, i32p, i32p]),
    "n1_image_digest": (c_int, [c_void_p, c_int64, c_void_p, c_int, c_void_p, c_void_p]),
    "n1_rope_index": (c_int, [i32p, c_int, i32p, c_int, c_int, i32p, i32p]),
    "n1_plan_rows_host": (c_int, [i32p, i32p, c_int, i32p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, i32p, i32p,
                                  c_int, i32p, i32p, i32p, i32p, i32p, i32p]),
    "n1_vit_window_index": (c_int, [i32p, c_int, c_int, c_int, i32p, i32p, i32p, i32p]),
    "n1_s2_set_latent_queries": (c_int, [c_void_p, c_void_p, c_void_p]),
    "n1_s2_train_workspace_bytes": (c_size_t, [c_void_p, c_void_p]),
    "n1_s2_train_forward": (c_int, [c_void_p, c_void_p, c_void_p, c_size_t, c_void_p, c_void_p, c_void_p]),
    "n1_s2_train_backward": (c_int, [c_void_p, c_void_p, c_void_p, c_size_t, c_void_p, c_void_p, c_void_p]),
    # frame preprocessing and System-2 image rows
    "n1_resize_plan_create": (c_int, [c_int, c_int, c_int, c_int, ctypes.POINTER(c_void_p), c_void_p]),
    "n1_resize_plan_destroy": (None, [c_void_p]),
    "n1_resize_workspace_bytes": (c_size_t, [c_void_p, c_int, c_int]),
    "n1_resize_rgb_u8": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "n1_resize_f32": (c_int, [c_void_p, c_void_p, c_int, c_float, c_float, c_void_p, c_void_p, c_size_t, c_void_p]),
    "n1_resize_coeffs": (c_int, [c_int, c_int, c_int, i32p, ctypes.POINTER(c_double), i32p, i32p]),
    "n1_vl_patchify_workspace_bytes": (c_size_t, [c_int]),
    "n1_vl_patchify": (c_int, [ctypes.POINTER(VlImage), c_int, c_void_p, c_void_p, c_int64, c_void_p, c_size_t, c_void_p]),
    # training: backward primitives
    "n1_op_transpose": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_int, c_int, c_void_p]),
    "n1_op_colsum": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_int, c_void_p]),
    "n1_op_norm_bwd": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p,
                               c_void_p, c_int, c_int, c_float, c_int, c_int, c_void_p]),
    "n1_op_act_fwd": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_void_p]),
    "n1_op_act_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_void_p]),
    "n1_op_swiglu_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_void_p]),
    "n1_op_rope_transposed": (c_int, [c_void_p, c_int, c_void_p, c_int64, c_int, c_int, c_void_p]),
    "n1_op_attention_bwd": (c_int, [c_void_p] * 8 + [c_int] * 12 + [c_void_p, c_void_p, c_int, c_int, c_int, c_float,
                                                                   c_void_p, c_int, c_void_p]),
    "n1_op_sgemm": (c_int, [c_void_p, c_int, c_int, c_void_p, c_int, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int,
                            c_void_p]),
    "n1_op_wgrad_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "n1_op_wgrad": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_int, c_void_p, c_size_t,
                            c_void_p]),
    "n1_op_scale_cols": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p, c_int, c_int64, c_int, c_void_p]),
    "n1_op_patchify_depth": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "n1_op_adamw": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_float, c_float, c_float, c_float,
                            c_float, c_int, c_void_p]),
    "n1_rgb_tokens_workspace_bytes": (c_size_t, [c_void_p, c_int]),
    "n1_rgb_tokens": (c_int, [c_void_p, c_void_p, c_size_t, c_void_p, c_void_p, c_int, c_void_p]),
    "n1_traj_to_actions": (c_int, [c_void_p, c_int, c_int, c_int, ctypes.c_double, ctypes.c_double, c_int, c_int, c_int,
                                   c_void_p, c_void_p, c_void_p, c_void_p]),
    "n1_traj_mean_path": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "n1_prof_enable": (None, [c_int]),
    "n1_prof_add": (None, [ctypes.c_int64, ctypes.c_int64]),
    "n1_prof_read": (c_int, [ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_double),
                             ctypes.POINTER(ctypes.c_int64), ctypes.POINTER(ctypes.c_int64)]),
    "n1_prof_read_shapes": (c_int, [ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_int64),
                                    ctypes.POINTER(ctypes.c_double), c_int]),
    "n1_op_gemm": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                           c_void_p, c_int, c_int, c_int, c_void_p]),
    "n1_op_ff_block": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_float, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                               c_int, c_int, c_void_p]),
    "n1_op_dec_sa_block": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_float, c_void_p, c_void_p, c_void_p, c_void_p,
                                   c_int, c_int, c_int, c_int, c_void_p]),
    "n1_op_dec_ca_block": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_float, c_void_p, c_void_p, c_void_p, c_void_p,
                                   c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "n1_op_layernorm": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_float, c_int,
                                c_void_p]),
    "n1_op_mod_norm": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_void_p, c_int, c_void_p, c_int,
                               ctypes.c_int64, c_int, c_float, c_int, c_void_p]),
    "n1_op_add": (c_int, [c_void_p, c_void_p, c_void_p, ctypes.c_int64, c_void_p]),
    "n1_op_action_embed": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, ctypes.c_int64, c_int, c_int, c_void_p]),
    "n1_op_cfg_euler": (c_int, [c_void_p, c_int, ctypes.c_int64, c_int, c_float, c_float, c_void_p, c_void_p]),
    "n1_op_attention_ex": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int,
                                   c_int, c_void_p, c_int, ctypes.c_int64, c_int, c_float, ctypes.POINTER(c_int), c_void_p]),
    "n1_op_attention": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int,
                                c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_float, c_void_p]),
    "n1_op_attention_cache": (c_int, [c_void_p, c_int, ctypes.c_int64, c_void_p, c_void_p, c_int, ctypes.c_int64, c_void_p,
                                      c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_float, c_void_p]),
    "n1_op_attention_cache_paged": (c_int, [c_void_p, c_int, ctypes.c_int64, c_void_p, c_void_p, c_int, ctypes.c_int64,
                                            c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                            c_int, c_float, c_void_p]),
}

OP_RGBD, OP_GOAL, OP_DENOISE = 1, 2, 3
ACT_NONE, ACT_GELU, ACT_RELU, ACT_SWIGLU, ACT_GELU_TANH, ACT_SILU = 0, 1, 2, 3, 4, 5


def lib():
    """Load the shared library (once).  Raises if it has not been built."""
    global _lib
    with _lock:
        if _lib is None:
            if not os.path.exists(LIB_PATH):
                raise ImportError(
                    "%s not found: build it with `python -m internnav_b200.build` (nvcc, sm_90a). "
                    "There is no CPU/PyTorch fallback for the n1b200 hot path." % LIB_PATH)
            L = ctypes.CDLL(LIB_PATH)
            for name, (res, args) in SYMBOLS.items():
                fn = getattr(L, name)
                fn.restype = res
                fn.argtypes = args
            _lib = L
    return _lib


def check(code):
    if code != 0:
        raise N1Error(code, lib().n1_last_error().decode("utf-8", "replace"))


def ptr(t):
    if t is None:
        return None
    assert t.is_cuda and t.is_contiguous(), "n1b200 takes contiguous CUDA tensors"
    return c_void_p(t.data_ptr())


def stream_ptr():
    return c_void_p(torch.cuda.current_stream().cuda_stream)


def dtype_code(t):
    if t.dtype == torch.float32:
        return 0
    if t.dtype == torch.bfloat16:
        return 1
    raise TypeError("n1b200 takes fp32 or bf16 tensors, got %s" % t.dtype)


def prof_enable(on):
    lib().n1_prof_enable(1 if on else 0)


def prof_read():
    """-> dict(gemm_ms, gemm_flops, gemm_launches, total_launches) since the last read."""
    a, b = ctypes.c_double(), ctypes.c_double()
    c, d = ctypes.c_int64(), ctypes.c_int64()
    check(lib().n1_prof_read(ctypes.byref(a), ctypes.byref(b), ctypes.byref(c), ctypes.byref(d)))
    return {"gemm_ms": a.value, "gemm_flops": b.value, "gemm_launches": c.value, "total_launches": d.value}


def prof_read_shapes(cap=256):
    """Per-shape GEMM timing of the last profiled region (call after prof_read): list of dict(M, N, K, count, ms)."""
    mnk = (ctypes.c_int32 * (3 * cap))()
    cnt = (ctypes.c_int64 * cap)()
    ms = (ctypes.c_double * cap)()
    n = lib().n1_prof_read_shapes(mnk, cnt, ms, cap)
    if n < 0:
        raise N1Error(n, lib().n1_last_error().decode("utf-8", "replace"))
    return [dict(M=mnk[3 * i], N=mnk[3 * i + 1], K=mnk[3 * i + 2], count=int(cnt[i]), ms=float(ms[i])) for i in range(n)]


# ------------------------------------------------------------------------------------------ kernel-level ops
def gemm(a, w, bias=None, gamma=None, residual=None, act=ACT_NONE, out_fp32=False, out=None):
    """out = epi(a @ w.T); a [M,K] bf16 (row stride allowed), w [N,K] bf16."""
    assert a.dtype == torch.bfloat16 and w.dtype == torch.bfloat16 and a.dim() == 2 and w.dim() == 2
    M, K = a.shape
    N = w.shape[0]
    n_out = N // 2 if act == ACT_SWIGLU else N
    if out is None:
        out = torch.empty(M, n_out, device=a.device, dtype=torch.float32 if out_fp32 else torch.bfloat16)
    assert a.stride(1) == 1 and w.stride(1) == 1 and out.stride(1) == 1
    check(lib().n1_op_gemm(c_void_p(a.data_ptr()), a.stride(0), c_void_p(w.data_ptr()), w.stride(0),
                           c_void_p(out.data_ptr()), out.stride(0), M, N, K, ptr(bias), ptr(gamma),
                           c_void_p(residual.data_ptr()) if residual is not None else None,
                           residual.stride(0) if residual is not None else 0, act, 1 if out_fp32 else 0, stream_ptr()))
    return out


def gemm_tile(a, w, out, bias=None, gamma=None, residual=None, act=ACT_NONE, rows_per_group=0, group_stride=0,
              group_offset=0, row_add=None, tile_n=0):
    """gemm() into a caller-owned view `out` (fp32 or bf16, any alignment) with the output row remap / row-add of the
    patch-embedding GEMMs and a forced tile width (tile_n 64 / 128 / 256; 0 = the dispatcher's choice).  For tests and
    scripts/bench_tiles.py: n1_test_gemm is exported but is not part of include/n1b200.h."""
    fn = lib().n1_test_gemm
    fn.restype = c_int
    fn.argtypes = [c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                   c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int, c_void_p]
    vp = lambda t: c_void_p(t.data_ptr()) if t is not None else None
    check(fn(vp(a), a.stride(0), vp(w), w.stride(0), vp(out), out.stride(0), a.shape[0], w.shape[0], a.shape[1],
             vp(bias), vp(gamma), vp(residual), residual.stride(0) if residual is not None else 0, act,
             1 if out.dtype == torch.float32 else 0, rows_per_group, group_stride, group_offset, vp(row_add), tile_n,
             stream_ptr()))
    return out


def layernorm(x, w, b=None, eps=1e-5, rms=False, out=None):
    assert x.dtype == torch.bfloat16 and x.dim() == 2 and x.stride(1) == 1
    y = torch.empty(x.shape, device=x.device, dtype=torch.bfloat16) if out is None else out
    assert y.stride(1) == 1 and y.shape == x.shape
    check(lib().n1_op_layernorm(c_void_p(x.data_ptr()), x.stride(0), c_void_p(y.data_ptr()), y.stride(0), ptr(w), ptr(b), x.shape[0],
                                x.shape[1], eps, 1 if rms else 0, stream_ptr()))
    return y


MOD_RMS_SCALE, MOD_LN_SCALE, MOD_GATED_RESIDUAL = 0, 1, 2


def mod_norm(x, w, mod, rows_per_group, eps, mode, residual=None, out=None):
    """Modulated / gated norms of the NextDiT block (csrc/nextdit_kernels.cu).  x bf16 [rows, D] (row stride allowed),
    w fp32 [D] or None, mod bf16 [groups, D] view (row stride allowed) or None."""
    assert x.dtype == torch.bfloat16 and x.dim() == 2 and x.stride(1) == 1
    if out is None:
        out = torch.empty(x.shape, device=x.device, dtype=torch.bfloat16)
    if mod is not None:
        assert mod.dtype == torch.bfloat16 and mod.stride(1) == 1 and mod.shape[1] == x.shape[1]
        assert mod.shape[0] * rows_per_group == x.shape[0]
    check(lib().n1_op_mod_norm(c_void_p(x.data_ptr()), x.stride(0), ptr(w), c_void_p(mod.data_ptr()) if mod is not None else None,
                               mod.stride(0) if mod is not None else 0, int(rows_per_group),
                               c_void_p(residual.data_ptr()) if residual is not None else None,
                               residual.stride(0) if residual is not None else 0, c_void_p(out.data_ptr()), out.stride(0),
                               x.shape[0], x.shape[1], float(eps), int(mode), stream_ptr()))
    return out


def add(a, b, out=None):
    assert a.dtype == torch.bfloat16 and b.dtype == torch.bfloat16 and a.is_contiguous() and b.is_contiguous() and a.shape == b.shape
    if out is None:
        out = torch.empty_like(a)
    check(lib().n1_op_add(ptr(a), ptr(b), ptr(out), a.numel(), stream_ptr()))
    return out


def action_embed(lat, w, b, pos, out=None):
    """lat fp32 [rows, 3], w fp32 [D, 3], b fp32 [D], pos fp32 [T, D] -> bf16 [rows, D]."""
    assert lat.dtype == torch.float32 and lat.is_contiguous() and lat.shape[-1] == 3
    rows, (T, D) = lat.numel() // 3, pos.shape
    if out is None:
        out = torch.empty(rows, D, device=lat.device, dtype=torch.bfloat16)
    check(lib().n1_op_action_embed(ptr(lat), ptr(w), ptr(b), ptr(pos), ptr(out), rows, T, D, stream_ptr()))
    return out


def cfg_euler(pred, n, cfg, scale, dt, lat):
    """lat fp32 [n, 3] <- bf16(lat + dt * guided(pred)); pred bf16 [(2 if cfg else 1) * n, >= 3]."""
    assert pred.dtype == torch.bfloat16 and pred.stride(1) == 1 and lat.dtype == torch.float32 and lat.is_contiguous()
    assert pred.shape[0] == (2 if cfg else 1) * n and lat.numel() == 3 * n
    check(lib().n1_op_cfg_euler(c_void_p(pred.data_ptr()), pred.stride(0), n, 1 if cfg else 0, float(scale), float(dt), ptr(lat),
                                stream_ptr()))
    return lat


def attention(q, k, v, heads_q, heads_kv, head_dim, batch, seq_q, seq_k, cu_q=None, cu_k=None, max_seq_q=0, kv_div=1,
              causal=False, scale=None):
    """q [rows_q, >=heads_q*hd], k/v [rows_k, >=heads_kv*hd] bf16 views with unit inner stride -> o [rows_q, heads_q*hd]."""
    assert q.dtype == torch.bfloat16 and q.stride(1) == 1 and k.stride(1) == 1 and v.stride(1) == 1
    o = torch.empty(q.shape[0], heads_q * head_dim, device=q.device, dtype=torch.bfloat16)
    if scale is None:
        scale = head_dim ** -0.5
    check(lib().n1_op_attention(c_void_p(q.data_ptr()), c_void_p(k.data_ptr()), c_void_p(v.data_ptr()), ptr(o),
                                q.stride(0), k.stride(0), v.stride(0), o.stride(0), heads_q, heads_kv, head_dim, batch,
                                seq_q, seq_k, ptr(cu_q), ptr(cu_k), max_seq_q, kv_div, 1 if causal else 0,
                                float(scale), stream_ptr()))
    return o


def attention_varlen(q, k, v, heads_q, heads_kv, head_dim, cu_seqlens, max_seq, causal=True, scale=None):
    """Var-len self-attention over packed rows (q / k / v: views with unit inner stride, `cu_seqlens` int32 [batch + 1]).
    -> (o [rows, heads_q * hd], used_tcgen05: whether the wgmma kernel ran)."""
    assert q.dtype == torch.bfloat16 and q.stride(1) == 1 and k.stride(1) == 1 and v.stride(1) == 1
    o = torch.empty(q.shape[0], heads_q * head_dim, device=q.device, dtype=torch.bfloat16)
    if scale is None:
        scale = head_dim ** -0.5
    used = c_int(0)
    check(lib().n1_op_attention_ex(c_void_p(q.data_ptr()), c_void_p(k.data_ptr()), c_void_p(v.data_ptr()), ptr(o),
                                   q.stride(0), k.stride(0), v.stride(0), o.stride(0), heads_q, heads_kv, head_dim,
                                   cu_seqlens.numel() - 1, ptr(cu_seqlens), int(max_seq), q.shape[0], 1 if causal else 0,
                                   float(scale), ctypes.byref(used), stream_ptr()))
    return o, bool(used.value)


ATTN_KERNELS = {1: "short", 2: "generic", 3: "wgmma"}


def attention_test(q, k, v, o, heads_q, heads_kv, head_dim, batch, seq_q=0, seq_k=0, cu_q=None, cu_k=None, max_seq_q=0,
                   kv_div=1, causal=False, scale=None, k_len=None, k_slot=0, k_row0=None, total_rows=0):
    """attention() with every AttnParams field into a caller-owned view `o` (q / k / v / o: views with unit inner stride;
    cu_q / cu_k / k_len / k_row0 int32 device tensors or None) -> the kernel that ran, as reported by the library's
    routing rule: ("short", 48, 16-key tiles, sequences per CTA), ("generic", head dim, 0, 1) or ("wgmma", 128, 0, 1).
    For tests: n1_test_attention is exported but is not part of include/n1b200.h."""
    for t in (q, k, v, o):
        assert t.dtype == torch.bfloat16 and t.stride(1) == 1
    fn = lib().n1_test_attention
    fn.restype = c_int
    fn.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int,
                   c_int, c_void_p, c_void_p, c_int, c_int, c_int, ctypes.c_float, c_void_p, c_int, c_void_p,
                   ctypes.c_int64, c_void_p, c_void_p]
    route = (c_int * 4)()
    vp = lambda t: c_void_p(t.data_ptr())
    check(fn(vp(q), vp(k), vp(v), vp(o), q.stride(0), k.stride(0), v.stride(0), o.stride(0), heads_q, heads_kv, head_dim,
             batch, seq_q, seq_k, ptr(cu_q), ptr(cu_k), int(max_seq_q), kv_div, 1 if causal else 0,
             float(head_dim ** -0.5 if scale is None else scale), ptr(k_len), int(k_slot), ptr(k_row0), int(total_rows),
             route, stream_ptr()))
    return ATTN_KERNELS[route[0]], route[1], route[2], route[3]


def attention_paged_test(q, k, v, o, heads_q, heads_kv, batch, seq_q, k_len, k_row0, pages, k_slot=0, scale=None):
    """The slotted-cache decode / latent-pass attention (attn_kernel, head_dim 128, causal) over a paged pool: sequence
    b's keys are its k_len[b] rows of the slotted view starting at k_row0[b] (a multiple of 64; or b * k_slot), whose row
    r lives at pool row pages[r // 64] * 64 + r % 64 of k / v.  q / o [batch * seq_q, >= heads * 128] views; k_len / k_row0
    / pages int32 device tensors.  For tests: n1_test_attention_paged is exported but not part of include/n1b200.h."""
    for t in (q, k, v, o):
        assert t.dtype == torch.bfloat16 and t.stride(1) == 1
    assert k.stride(0) == v.stride(0)
    fn = lib().n1_test_attention_paged
    fn.restype = c_int
    fn.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int,
                   c_void_p, c_void_p, ctypes.c_float, c_void_p]
    vp = lambda t: c_void_p(t.data_ptr())
    check(fn(vp(q), vp(k), vp(v), vp(o), q.stride(0), k.stride(0), o.stride(0), heads_q, heads_kv, batch, seq_q,
             ptr(k_len), int(k_slot), ptr(k_row0), ptr(pages), float(128 ** -0.5 if scale is None else scale),
             stream_ptr()))


def attention_cache(q, k, v, heads_q, heads_kv, cu_q, ctx, row0, max_chunk, scale=None, out=None, pages=None):
    """Chunk attention over a slotted K/V cache (head_dim 128): q [rows, >=heads_q*128] packed chunk rows (sequence b at
    cu_q[b] .. cu_q[b + 1]), k / v [kv_rows, heads_kv*128] cache rows (sequence b's keys at row0[b] .. row0[b] + ctx[b] +
    n_b - 1), cu_q / ctx / row0 int32 device tensors -> o [rows, heads_q*128] bf16, bottom-right causal.  `out` may be
    a view with a wider row stride."""
    assert q.dtype == k.dtype == v.dtype == torch.bfloat16 and q.stride(1) == 1 and k.stride(1) == 1 and v.stride(1) == 1
    assert k.stride(0) == v.stride(0) and k.shape[0] == v.shape[0]
    for t in (cu_q, ctx, row0):
        assert t.dtype == torch.int32 and t.is_cuda and t.is_contiguous()
    o = torch.empty(q.shape[0], heads_q * 128, device=q.device, dtype=torch.bfloat16) if out is None else out
    assert o.dtype == torch.bfloat16 and o.stride(1) == 1 and o.is_cuda
    scale = float(128 ** -0.5 if scale is None else scale)
    if pages is None:
        check(lib().n1_op_attention_cache(c_void_p(q.data_ptr()), q.stride(0), q.shape[0], c_void_p(k.data_ptr()),
                                          c_void_p(v.data_ptr()), k.stride(0), k.shape[0], c_void_p(o.data_ptr()), o.stride(0), ptr(cu_q),
                                          ptr(ctx), ptr(row0), cu_q.numel() - 1, int(max_chunk), heads_q, heads_kv,
                                          scale, stream_ptr()))
        return o
    assert pages.dtype == torch.int32 and pages.is_cuda and pages.is_contiguous()
    check(lib().n1_op_attention_cache_paged(c_void_p(q.data_ptr()), q.stride(0), q.shape[0], c_void_p(k.data_ptr()),
                                            c_void_p(v.data_ptr()), k.stride(0), k.shape[0], c_void_p(o.data_ptr()),
                                            o.stride(0), ptr(cu_q), ptr(ctx), ptr(row0), ptr(pages), cu_q.numel() - 1,
                                            int(max_chunk), heads_q, heads_kv, scale, stream_ptr()))
    return o


def ff_block(x, ln_w, ln_b, w1, b1, w2, b2, eps=1e-5, out=None):
    """out = x + gelu(LayerNorm(x) @ w1.T + b1) @ w2.T + b2 (NavDP decoder FF block, one fused kernel)."""
    assert x.dtype == torch.bfloat16 and x.shape[1] == 384 and w1.shape == (1536, 384) and w2.shape == (384, 1536)
    assert w1.is_contiguous() and w2.is_contiguous() and x.stride(1) == 1
    if out is None:
        out = torch.empty(x.shape[0], 384, device=x.device, dtype=torch.bfloat16)
    check(lib().n1_op_ff_block(c_void_p(x.data_ptr()), x.stride(0), ptr(ln_w), ptr(ln_b), eps, ptr(w1), ptr(b1), ptr(w2),
                               ptr(b2), c_void_p(out.data_ptr()), out.stride(0), x.shape[0], stream_ptr()))
    return out


def dec_sa_block(x, ln_w, ln_b, w_qkv, b_qkv, w_o, b_o, B, Ns, T, causal=True, eps=1e-5):
    """In place: x += w_o-projection of per-trajectory MHA(LayerNorm(x) @ w_qkv.T + b_qkv) + b_o (NavDP decoder
    self-attention sublayer, one fused kernel).  x bf16 [B * Ns * T, 384] view (row stride allowed)."""
    assert x.dtype == torch.bfloat16 and x.shape == (B * Ns * T, 384) and x.stride(1) == 1
    assert w_qkv.shape == (1152, 384) and w_o.shape == (384, 384)
    check(lib().n1_op_dec_sa_block(c_void_p(x.data_ptr()), x.stride(0), ptr(ln_w), ptr(ln_b), float(eps), ptr(w_qkv),
                                   ptr(b_qkv), ptr(w_o), ptr(b_o), B, Ns, T, 1 if causal else 0, stream_ptr()))
    return x


def dec_ca_block(x, ln_w, ln_b, w_q, b_q, w_o, b_o, kv, mtok, B, Ns, T, eps=1e-5):
    """In place: x += w_o-projection of MHA(LayerNorm(x) @ w_q.T + b_q, K_e, V_e) + b_o (NavDP decoder cross-attention
    sublayer, one fused kernel).  kv bf16 view [B * mtok, >= 768] (row stride allowed): K in columns 0..383, V in 384..767."""
    assert x.dtype == torch.bfloat16 and x.shape == (B * Ns * T, 384) and x.stride(1) == 1
    assert w_q.shape == (384, 384) and w_o.shape == (384, 384) and kv.shape[0] == B * mtok and kv.stride(1) == 1
    check(lib().n1_op_dec_ca_block(c_void_p(x.data_ptr()), x.stride(0), ptr(ln_w), ptr(ln_b), float(eps), ptr(w_q), ptr(b_q),
                                   ptr(w_o), ptr(b_o), c_void_p(kv.data_ptr()), kv.stride(0), mtok, B, Ns, T, stream_ptr()))
    return x
