"""The warp-specialised tensor-core kernels that reallocate registers (setmaxnreg: producer warpgroup 40, consumer
warpgroups 232) must compile for sm_90a without a byte of register spill.  The 256-wide GEMM tile, the FF block and the
decoder attention blocks only fit because of that reallocation, and a spill in their main loops is a silent slowdown no
other test would see.  attn_small_kernel shares its attention core (dec_tile.cuh) with the decoder attention blocks, so a
change made for those is checked against it too."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _nvcc():
    from internnav_b200 import build
    return build.NVCC if os.path.exists(build.NVCC) else shutil.which("nvcc")


@pytest.mark.skipif(_nvcc() is None, reason="nvcc not installed")
@pytest.mark.parametrize("src,kernel,entries", [("gemm_wgmma.cu", "gemm_kernel", 3), ("ff_block.cu", "ff_block_kernel", 1),
                                                ("dec_attn_block.cu", "dec_attn_kernel", 2),
                                                ("attention.cu", "attn_small_kernel", 4)])
def test_kernels_compile_without_spills(tmp_path, src, kernel, entries):
    from internnav_b200 import build
    cmd = [_nvcc()] + build.FLAGS + ["-c", os.path.join(build.CSRC, src), "-o", str(tmp_path / "k.o")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    # ptxas -v: "Compiling entry function '<mangled>'" ... "N bytes stack frame, N bytes spill stores, N bytes spill loads"
    found = re.findall(r"Function properties for (\S*%s\S*)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads" % kernel, r.stderr)
    assert len(found) == entries, (len(found), r.stderr[-2000:])
    for name, stack, st, ld in found:
        assert (int(stack), int(st), int(ld)) == (0, 0, 0), "%s: %s bytes stack, %s / %s bytes spilled" % (name, stack, st, ld)
    assert "wgmma.mma_async instructions are serialized" not in r.stderr
