"""The wgmma GEMM compiles one epilogue kind per kernel instance (csrc/gemm_wgmma.cu): gemm_kernel<BN> carries the linear
(bias / layer-scale / residual) and SwiGLU kinds with TMA stores, gemm_act_kernel<BN, act> one activation each, and
gemm_act_kernel<BN, KIND_GENERAL> the direct-store path.  When every kind was inlined at each accumulator position, a plain
tile's epilogue walked 100 - 200 KB of machine code; these tests hold the System-2 entries to at most half of that size and
every instance to 0 bytes of spill, and check the swizzled staging layout of the bf16 output tile against the tensor
map's swizzle and the shared-memory banks."""
import os
import re
import shutil
import subprocess

import pytest

# SASS instructions (16 bytes each) of gemm_kernel<BN> when every epilogue kind was inlined in it
UNSPLIT_SASS = {128: 7208, 256: 13840}
# what the linear / SwiGLU entries may grow to
SASS_BOUND = {128: 3000, 256: 5200}
ACT_GELU, ACT_RELU, ACT_GELU_TANH, ACT_SILU, KIND_GENERAL = 1, 2, 4, 5, 8


def _nvcc():
    from internnav_b200 import build
    return build.NVCC if os.path.exists(build.NVCC) else shutil.which("nvcc")


def _cuobjdump():
    nvcc = _nvcc()
    if nvcc is None:
        return None
    path = os.path.join(os.path.dirname(nvcc), "cuobjdump")
    return path if os.path.exists(path) else shutil.which("cuobjdump")


@pytest.fixture(scope="module")
def gemm_object(tmp_path_factory):
    from internnav_b200 import build
    obj = str(tmp_path_factory.mktemp("gemm") / "gemm_wgmma.o")
    r = subprocess.run([_nvcc()] + build.FLAGS + ["-c", os.path.join(build.CSRC, "gemm_wgmma.cu"), "-o", obj],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return obj, r.stderr


def _instance(name):
    """mangled entry -> (BN, kind) with kind None for gemm_kernel<BN>, or None for anything else"""
    m = re.search(r"gemm_kernelILi(\d+)EE", name)
    if m:
        return int(m.group(1)), None
    m = re.search(r"gemm_act_kernelILi(\d+)ELi(\d+)EE", name)
    return (int(m.group(1)), int(m.group(2))) if m else None


@pytest.mark.skipif(_nvcc() is None or _cuobjdump() is None, reason="nvcc / cuobjdump not installed")
def test_every_instance_is_spill_free(gemm_object):
    _, log = gemm_object
    found = re.findall(r"Function properties for (\S+)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", log)
    inst = {_instance(name): (int(a), int(b), int(c)) for name, a, b, c in found if _instance(name)}
    want = {(bn, kind) for bn in (64, 128, 256) for kind in (None, ACT_GELU, ACT_RELU, ACT_GELU_TANH, ACT_SILU, KIND_GENERAL)}
    assert set(inst) == want, sorted(inst)
    for key, spill in inst.items():
        assert spill == (0, 0, 0), "%s: %s bytes stack / spill stores / spill loads" % (key, spill)
    assert "wgmma.mma_async instructions are serialized" not in log


@pytest.mark.skipif(_nvcc() is None or _cuobjdump() is None, reason="nvcc / cuobjdump not installed")
def test_system2_entries_are_compact(gemm_object):
    obj, _ = gemm_object
    r = subprocess.run([_cuobjdump(), "-sass", obj], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    counts, name = {}, None
    for line in r.stdout.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1)
            counts[name] = 0
        elif name and re.match(r"\s+/\*[0-9a-f]+\*/\s", line):
            counts[name] += 1
    sizes = {_instance(n)[0]: c for n, c in counts.items() if _instance(n) and _instance(n)[1] is None}
    assert sorted(sizes) == [64, 128, 256], sorted(counts)
    for bn, bound in SASS_BOUND.items():
        assert 2 * bound <= UNSPLIT_SASS[bn]
        assert sizes[bn] <= bound, "gemm_kernel<%d>: %d SASS instructions (bound %d)" % (bn, sizes[bn], bound)


def _swizzle(offset, span):
    """byte offset -> where TMA's 32 / 64 / 128-byte swizzle puts it: 16-byte chunk bits XOR the bits from 128 up"""
    bits = {32: 1, 64: 2, 128: 3}[span]
    return offset ^ (((offset >> 7) & ((1 << bits) - 1)) << 4)


def test_staging_layout_matches_the_swizzle_and_is_bank_conflict_free():
    # the epilogue's staging store addresses (gemm_wgmma.cu), lane = 4 r + quad, h = row half, j = 8-column group
    plain = lambda r, j, quad: r * 64 + (((j ^ (r >> 1)) & 3) << 4) + quad * 4  # 4-byte stores, 64-byte rows
    swiglu = lambda r, j, quad: r * 32 + ((((j >> 1) ^ (r >> 2)) & 1) << 4) + (j & 1) * 8 + quad * 2  # 2-byte, 32-byte
    for j in range(4):
        for h in range(2):
            rows = [(lane >> 2) + 8 * h for lane in range(32)]
            quads = [lane & 3 for lane in range(32)]
            p = [plain(r, j, q) for r, q in zip(rows, quads)]
            s = [swiglu(r, j, q) for r, q in zip(rows, quads)]
            # the same bytes the tensor map reads for row r, column 8 j + 2 quad (SwiGLU: 4 j + quad)
            assert p == [_swizzle(r * 64 + j * 16 + q * 4, 64) for r, q in zip(rows, quads)]
            assert s == [_swizzle(r * 32 + j * 8 + q * 2, 32) for r, q in zip(rows, quads)]
            # one warp's store: 32 distinct banks; SwiGLU: two lanes per 4-byte word, 16 distinct banks
            assert len({a // 4 % 32 for a in p}) == 32
            words = {a // 4 for a in s}
            assert len(words) == 16 and len({w % 32 for w in words}) == 16
            # unswizzled, the same stores conflicted 4-way (plain) and 2-way (SwiGLU)
            assert len({(r * 64 + j * 16 + q * 4) // 4 % 32 for r, q in zip(rows, quads)}) == 8
            assert len({(r * 32 + j * 8 + q * 2) // 4 % 32 for r, q in zip(rows, quads)}) == 8
