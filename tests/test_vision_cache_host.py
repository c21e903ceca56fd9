"""Host-side rules of the System-2 vision-feature pool: the pool's bookkeeping (keys, LRU order, the current call's
entries kept, free-list reuse, a pool too small for one call), the share of the reference's history frames a pool
serves, the argument checks of the entry points that read and write pool rows, and the register budget of the changed
kernels."""
import ctypes
import os
import re
import subprocess
from types import SimpleNamespace

import numpy as np
import pytest
import torch


def _pool(rows, width=8):
    from internnav_b200.qwen import ImageFeaturePool
    return ImageFeaturePool(SimpleNamespace(cfg={"v_out": width}, device=torch.device("cpu")), rows)


def test_pool_keys_include_the_grid():
    p = _pool(100)
    a, b = (7, 1, 4, 4), (7, 1, 2, 8)    # one digest, two grids: two entries
    rows, new = p.assign([a, b], [4, 4])
    assert new == {a, b} and len(p) == 2 and p.free_rows == 92
    assert sorted(np.concatenate(rows).tolist()) == list(range(8))
    rows2, new2 = p.assign([b, a], [4, 4])
    assert new2 == set() and [r.tolist() for r in rows2] == [rows[1].tolist(), rows[0].tolist()]
    assert p.bytes == 100 * 8 * 2


def test_pool_lru_order_pinning_and_free_list_reuse():
    p = _pool(12)
    keys = [(i, 1, 2, 2) for i in range(4)]
    for k in keys[:3]:
        p.assign([k], [1 * 4])          # three entries of 4 rows fill the pool
    assert p.free_rows == 0 and p.keys() == keys[:3]
    p.assign([keys[0]], [4])            # a hit becomes the most recently used
    assert p.keys() == [keys[1], keys[2], keys[0]]
    old = p.rows_of(keys[1])
    rows, new = p.assign([keys[0], keys[3]], [4, 4])   # needs 4 rows: the oldest entry outside the call goes
    assert new == {keys[3]} and keys[1] not in p and p.keys() == [keys[2], keys[0], keys[3]]
    assert sorted(rows[1].tolist()) == sorted(old)     # the evicted rows are reused
    # the call uses keys[2] and keys[3] and needs 4 new rows: keys[0] (older than keys[3] but unused) goes, not keys[2]
    rows, new = p.assign([keys[2], keys[1], keys[3]], [4, 4, 4])
    assert new == {keys[1]} and keys[0] not in p and set(p.keys()) == {keys[1], keys[2], keys[3]}
    assert sorted(np.concatenate(rows).tolist()) == list(range(12))
    # rows of a discarded entry return to the free list
    p.discard([keys[1]])
    assert keys[1] not in p and p.free_rows == 4


def test_pool_rows_allocated_one_at_a_time():
    """Freed rows that are not adjacent still serve a larger image: there is no fragmentation."""
    p = _pool(6)
    for i in range(6):
        p.assign([(i, 1, 2, 2)], [1])
    p.discard([(1, 1, 2, 2), (3, 1, 2, 2), (5, 1, 2, 2)])
    rows, _ = p.assign([(9, 1, 2, 6)], [3])
    assert sorted(rows[0].tolist()) == [1, 3, 5]


def test_pool_too_small_for_one_call():
    p = _pool(10)
    with pytest.raises(ValueError, match="needs 12 rows"):
        p.assign([(1, 1, 4, 4), (2, 1, 4, 4), (3, 1, 4, 4)], [4, 4, 4])
    rows, new = p.assign([(1, 1, 4, 4), (1, 1, 4, 4), (2, 1, 4, 4)], [4, 4, 4])  # a repeated image counts once
    assert len(new) == 2 and rows[0] is rows[1]
    with pytest.raises(ValueError):
        _pool(0)


def history_calls(n_frames, gap, num_history=8):
    """Images of the fresh System-2 calls of one episode, as frame indices: a call every `gap` frames, each with the
    reference's history pick np.unique(np.linspace(0, n - 1, num_history)) and the current frame."""
    calls = []
    for t in range(0, n_frames, gap):
        hist = [] if t == 0 else np.unique(np.linspace(0, t - 1, num_history, dtype=np.int32)).tolist()
        calls.append((hist, t))
    return calls


@pytest.mark.parametrize("gap", [2, 4, 8])
def test_history_hits_match_a_set_count(gap):
    """An unbounded pool serves exactly the history frames some earlier call encoded; a bounded one at most that."""
    calls = history_calls(500, gap)
    seen, want, picks = set(), 0, 0
    for hist, cur in calls:
        want += sum(1 for f in hist if f in seen)
        picks += len(hist)
        seen.update(hist + [cur])
    for rows, exact in ((10 ** 6, True), (40 * 4, False)):
        p, got = _pool(rows), 0
        for hist, cur in calls:
            keys = [(f, 1, 4, 4) for f in hist + [cur]]
            _, new = p.assign(keys, [4] * len(keys))
            got += sum(1 for k in keys[:-1] if k not in new)
        assert (got == want) if exact else (0 < got <= want), (got, want)
    share = want / picks
    print("gap %d: %.0f %% of %d history picks already encoded" % (gap, 100 * share, picks))
    assert share > {2: 0.8, 4: 0.65, 8: 0.45}[gap]


def test_vit_and_generate_refuse_bad_arguments():
    """The checks that need no device: a null handle, plan or pixels, or too many eos ids, is refused before anything
    runs."""
    from internnav_b200 import _lib
    L = _lib.lib()
    fake = ctypes.c_void_p(1 << 20)
    rows = (ctypes.c_int32 * 4)(0, 1, 2, 3)
    toks, lens = (ctypes.c_int32 * 4)(), (ctypes.c_int32 * 1)()
    assert L.n1_qwen_vit(None, fake, fake, 1, fake, fake, 8, rows, 4, None) == -2
    assert b"null handle" in L.n1_last_error()
    assert L.n1_qwen_vit(fake, None, fake, 1, fake, fake, 8, rows, 4, None) == -2
    assert L.n1_qwen_vit(fake, fake, fake, 1, None, fake, 8, rows, 4, None) == -2
    assert L.n1_llm_generate(None, fake, fake, 1, fake, 8, rows, 4, None, 0, 0, toks, lens, None, None, None) == -2
    assert L.n1_llm_generate(fake, None, fake, 1, fake, 8, rows, 4, None, 0, 0, toks, lens, None, None, None) == -2
    assert b"null handle / plan" in L.n1_last_error()
    assert L.n1_llm_generate(fake, fake, fake, 1, fake, 8, rows, 4, None, 5, 0, toks, lens, None, None, None) == -2
    assert b"eos" in L.n1_last_error()


def test_row_kernels_compile_without_spills(tmp_path):
    from internnav_b200 import build
    if not os.path.exists(build.NVCC):
        pytest.skip("nvcc not installed")
    cmd = [build.NVCC] + build.FLAGS + ["-c", os.path.join(build.CSRC, "s2_kernels.cu"), "-o", str(tmp_path / "k.o")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    for kernel in ("gather_rows_kernel", "build_embeds_kernel"):
        found = re.findall(r"Function properties for (\S*%s\S*)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                           r"(\d+) bytes spill loads" % kernel, r.stderr)
        assert len(found) == 1, (kernel, r.stderr[-2000:])
        assert tuple(int(v) for v in found[0][1:]) == (0, 0, 0), found
