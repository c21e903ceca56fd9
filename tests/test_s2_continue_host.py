"""Host-side rules of continuing a System-2 conversation on its K/V cache: which prefix of a new prompt a cache may
serve, the mRoPE positions of that prefix, the plan's row bookkeeping, and the chunk attention kernel's register budget."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

IMG = 151655


def _prompt(rng, pre, n_tok, post):
    return rng.integers(0, 151643, pre).tolist() + [151652] + [IMG] * n_tok + [151653] + rng.integers(0, 151643, post).tolist()


def test_reuse_length_rules():
    from internnav_b200.qwen import image_spans, reuse_length
    rng = np.random.Generator(np.random.PCG64(0))
    p1 = _prompt(rng, 5, 16, 4) + [1, 2, 3]                 # one 8 x 8 image at tokens 6 .. 21
    grids = [(1, 8, 8)]
    spans = image_spans(p1, grids)
    assert spans == [(6, 16)]
    cached = {6: (16, 111)}
    p2 = p1 + [9, 9] + [151652] + [IMG] * 4 + [151653] + [7]
    imgs = [(6, 16, 111), (len(p1) + 3, 4, 222)]
    assert [(s, n) for s, n, _ in imgs] == image_spans(p2, grids + [(1, 4, 4)])
    # whole previous conversation reused; the new image lies after it
    assert reuse_length(p1, cached, p2, imgs, cap=100, need=60) == len(p1)
    # token mismatch after position 3 -> cut there
    p3 = p1[:3] + [p1[3] + 1] + p1[4:]
    assert reuse_length(p1, cached, p3 + [5], [(6, 16, 111)], 100, 60) == 3
    # image digest mismatch -> cut at the image's first token
    assert reuse_length(p1, {6: (16, 999)}, p2, imgs, 100, 60) == 6
    # a prefix that would end inside an image is cut back to the image's start
    assert reuse_length(p1[:10], cached, p2, imgs, 100, 60) == 6
    # capacity overflow: nothing is reused (the conversation does not fit the slot)
    assert reuse_length(p1, cached, p2, imgs, cap=59, need=60) == 0
    # never the whole prompt: its last row must be prefilled (its logits start the decode)
    assert reuse_length(p2, {6: (16, 111), len(p1) + 3: (4, 222)}, p2, imgs, 100, 60) == len(p2) - 1


def test_handle_excludes_traj_rows_and_goes_stale():
    """A cache covers prompt + generated ids (never the n_query TRAJ rows of the latent pass) and is empty once another
    call rewrote its slot."""
    from internnav_b200.qwen import KVCache

    class _Pool:
        version = [0, 0]
    pool = _Pool()
    h = KVCache(pool, 1, [1, 2, 3, 4], {})
    assert len(h) == 4
    pool.version[1] += 1
    assert len(h) == 0


def test_mrope_positions_continue():
    """n1_rope_index over the look-down prompt, restricted to the reused prefix, equals the positions the previous call
    used: the prompt's own positions, then len + delta for each decoded token on all three axes."""
    from internnav_b200 import _lib
    L = _lib.lib()
    rng = np.random.Generator(np.random.PCG64(1))
    grids = [1, 8, 12, 1, 4, 8]
    p1 = _prompt(rng, 4, 24, 3)
    p1 = p1[:-3] + [151652] + [IMG] * 8 + [151653] + p1[-3:]
    gen = [11, 12, 13, 151645]
    p2 = p1 + gen + [198] + [151652] + [IMG] * 20 + [151653] + [5, 6]
    grids2 = grids + [1, 8, 10]

    def rope(ids, g):
        out = (ctypes.c_int32 * (3 * len(ids)))()
        d = ctypes.c_int32()
        assert L.n1_rope_index((ctypes.c_int32 * len(ids))(*ids), len(ids), (ctypes.c_int32 * len(g))(*g), len(g) // 3, 2,
                               out, ctypes.byref(d)) == 0, L.n1_last_error()
        return np.array(out).reshape(3, len(ids)), d.value
    pos1, delta = rope(p1, grids)
    pos2, _ = rope(p2, grids2)
    n1 = len(p1)
    assert (pos2[:, :n1] == pos1).all()
    for i in range(len(gen)):
        assert (pos2[:, n1 + i] == n1 + i + delta).all()


def _plan_rows(prompts, grids, max_new, reused=None, slots=None, pool=(0, 0), n_query=4):
    from internnav_b200 import _lib
    L = _lib.lib()
    i32 = ctypes.c_int32
    flat = [t for p in prompts for t in p]
    g = [v for gr in grids for v in gr]
    B, cap_rows = len(prompts), len(flat)
    n, cu, kind, src, dest, kl = i32(), (i32 * (B + 1))(), (i32 * cap_rows)(), (i32 * cap_rows)(), (i32 * cap_rows)(), (i32 * B)()
    arr = lambda v: None if v is None else (i32 * len(v))(*v)
    rc = L.n1_plan_rows_host(arr(flat), arr([len(p) for p in prompts]), B, (i32 * max(1, len(g)))(*g), len(g) // 3, 2,
                             152064, n_query, max_new, pool[0], pool[1], arr(reused), arr(slots), cap_rows, ctypes.byref(n),
                             cu, kind, src, dest, kl)
    if rc != 0:
        raise RuntimeError(L.n1_last_error().decode())
    r = n.value
    return list(cu), list(kind)[:r], list(src)[:r], list(dest)[:r], list(kl)


def test_plan_rows_mixed_batch():
    """A batch of a fresh and a continued sequence: only the continued one's suffix is planned, image features are
    numbered over the suffix images alone, K/V rows land in each sequence's pool slot, and the keys cover the whole prompt."""
    rng = np.random.Generator(np.random.PCG64(2))
    p0 = _prompt(rng, 3, 4, 2)                                   # fresh: one 4 x 4 image (4 tokens) at 4 .. 7
    p1 = _prompt(rng, 2, 16, 3) + [151652] + [IMG] * 4 + [151653] + [9]   # images at 3 .. 18 and 25 .. 28
    grids = [(1, 4, 4), (1, 8, 8), (1, 4, 4)]
    c1 = 24                                                      # reuse through the first image and the text after it
    cu, kind, src, dest, kl = _plan_rows([p0, p1], grids, 5, reused=[0, c1], slots=[2, 0], pool=(3, 100))
    n0, n1 = len(p0), len(p1) - c1
    assert cu == [0, n0, n0 + n1]
    assert kind == [1 if t == IMG else 0 for t in p0] + [1 if t == IMG else 0 for t in p1[c1:]]
    img_rows = [i for i, k in enumerate(kind) if k == 1]
    assert [src[i] for i in img_rows] == list(range(4 + 4))     # 4 features of p0's image, then 4 of p1's second image
    assert [src[i] for i, k in enumerate(kind) if k == 0] == [t for t in p0 + p1[c1:] if t != IMG]
    assert dest == [200 + i for i in range(n0)] + [c1 + i for i in range(n1)]
    assert kl == [len(p0), len(p1)]
    # the same prompts uncached: every row, slots b * (max_len + max_new + n_query)
    cu, kind, _, dest, kl = _plan_rows([p0, p1], grids, 5)
    slot = len(p1) + 5 + 4
    assert cu == [0, len(p0), len(p0) + len(p1)] and dest == list(range(len(p0))) + [slot + i for i in range(len(p1))]
    # a reused prefix may not end inside an image, nor a conversation overflow its slot
    with pytest.raises(RuntimeError, match="inside an image"):
        _plan_rows([p0, p1], grids, 5, reused=[0, 10], slots=[2, 0], pool=(3, 100))
    with pytest.raises(RuntimeError, match="capacity"):
        _plan_rows([p0, p1], grids, 80, reused=[0, c1], slots=[2, 0], pool=(3, 100))


def _nvcc():
    from internnav_b200 import build
    return build.NVCC if os.path.exists(build.NVCC) else shutil.which("nvcc")


@pytest.mark.skipif(_nvcc() is None, reason="nvcc not installed")
def test_attention_cache_kernel_compiles_without_spills(tmp_path):
    from internnav_b200 import build
    cmd = [_nvcc()] + build.FLAGS + ["-c", os.path.join(build.CSRC, "attention_cache_wgmma.cu"), "-o", str(tmp_path / "k.o")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    found = re.findall(r"Function properties for (\S*attn_cache_kernel\S*)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes "
                       r"spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(found) == 1, r.stderr[-2000:]
    assert tuple(int(v) for v in found[0][1:]) == (0, 0, 0), found
    assert "wgmma.mma_async instructions are serialized" not in r.stderr
