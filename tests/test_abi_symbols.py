"""The shared library loads without a GPU and exports every function include/n1b200.h declares."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_every_declared_symbol_is_exported():
    from internnav_b200 import _lib
    L = _lib.lib()
    with open(os.path.join(ROOT, "include", "n1b200.h")) as fh:
        src = re.sub(r"/\*.*?\*/", "", fh.read(), flags=re.S)
    names = sorted(set(re.findall(r"\b(n1_[a-z0-9_]+)\s*\(", src)))
    assert len(names) >= 30
    for n in names:
        assert hasattr(L, n), "missing export: " + n
    assert L.n1_version().decode().startswith("n1b200")


def test_no_gpu_fails_loudly():
    """Compute entry points must not fall back to anything when no sm_90 device is usable."""
    import torch
    from internnav_b200 import _lib
    L = _lib.lib()
    if torch.cuda.is_available():
        return
    h = ctypes.c_void_p()
    rc = L.n1_create(ctypes.byref(h), 0)
    assert rc != 0 and b"no CUDA device" in L.n1_last_error() or rc != 0


def test_ddpm_tables_match_oracle():
    import numpy as np
    from internnav_b200 import _lib
    from oracle import ddpm
    L = _lib.lib()
    for K in (20, 50):
        buf = (ctypes.c_float * (K * 5))()
        assert L.n1_ddpm_tables(K, buf) == 0
        mine = np.asarray(list(buf), dtype=np.float32).reshape(K, 5)
        ref = ddpm.DDPMScheduler(num_train_timesteps=K).coef_table()
        assert np.allclose(mine, ref, rtol=2e-5, atol=1e-7), np.abs(mine - ref).max()


def test_host_planner_error_behaviour():
    """Integer planners reject inconsistent prompts with an error code and message (no exception crosses the ABI)."""
    from internnav_b200 import _lib
    L = _lib.lib()
    ids = [1, 2, 151652] + [151655] * 10 + [151653, 5]          # 10 image pads
    a = (ctypes.c_int32 * len(ids))(*ids)
    out = (ctypes.c_int32 * (3 * len(ids)))()
    d = ctypes.c_int32()
    g_ok = (ctypes.c_int32 * 3)(1, 4, 10)                        # 1 x 4 x 10 patches -> 10 merged tokens
    assert L.n1_rope_index(a, len(ids), g_ok, 1, 2, out, ctypes.byref(d)) == 0
    g_bad = (ctypes.c_int32 * 3)(1, 8, 10)                       # 20 merged tokens: more than the prompt holds
    rc = L.n1_rope_index(a, len(ids), g_bad, 1, 2, out, ctypes.byref(d))
    assert rc != 0 and len(L.n1_last_error()) > 0
    rc = L.n1_rope_index(a, len(ids), g_ok, 0, 2, out, ctypes.byref(d))   # placeholder without a grid row
    assert rc != 0 and b"image_grid_thw" in L.n1_last_error()
    # odd grids cannot be merged 2 x 2
    bad = (ctypes.c_int32 * 3)(1, 5, 10)
    n = ctypes.c_int32()
    assert L.n1_vit_window_index(bad, 1, 2, 4, None, None, ctypes.byref(n), None) != 0
    # text-only prompt: positions are 0..n-1 on all three streams, delta 0
    t = (ctypes.c_int32 * 6)(7, 8, 9, 10, 11, 12)
    o = (ctypes.c_int32 * 18)()
    assert L.n1_rope_index(t, 6, g_ok, 0, 2, o, ctypes.byref(d)) == 0
    assert list(o) == list(range(6)) * 3 and d.value == 0


def test_null_arguments_are_errors():
    from internnav_b200 import _lib
    L = _lib.lib()
    assert L.n1_ddpm_tables(0, None) != 0
    assert L.n1_workspace_bytes(None, 1, 1, 1, 1) == 0 and b"null handle" in L.n1_last_error()
    L.n1_destroy(None)  # no-op


def test_every_declared_symbol_is_bound_with_its_arity():
    """Every function include/n1b200.h declares has a ctypes binding that passes as many arguments as the header declares
    (a mismatch would corrupt the call silently)."""
    import re
    from internnav_b200 import _lib
    L = _lib.lib()
    with open(os.path.join(ROOT, "include", "n1b200.h")) as fh:
        src = re.sub(r"/\*.*?\*/", "", fh.read(), flags=re.S)
    decl = {}
    for m in re.finditer(r"\b(n1_[a-z0-9_]+)\s*\(([^;{]*?)\)\s*;", src, flags=re.S):
        args = m.group(2).strip()
        decl[m.group(1)] = 0 if args in ("", "void") else args.count(",") + 1
    assert len(decl) >= 80 and set(decl) == set(_lib.SYMBOLS), set(decl) ^ set(_lib.SYMBOLS)
    for name, n in decl.items():
        fn = getattr(L, name)
        assert fn.argtypes is not None, "%s has no binding" % name
        assert len(fn.argtypes) == n, "%s: header declares %d arguments, binding passes %d" % (name, n, len(fn.argtypes))
