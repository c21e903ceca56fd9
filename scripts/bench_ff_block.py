"""Micro-benchmark of the NavDP decoder FF block at the benchmark row count (65536 = 64 envs x 32 samples x T 32):
LayerNorm + FF1(GELU) + FF2(residual) as three library kernels vs the one-kernel FF block (ff_block.cu), CUDA events,
L2 flushed between repetitions.  Prints one JSON line."""
import json
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from internnav_b200 import _lib as L  # noqa: E402


def timed(fn, reps=20):
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    for _ in range(3):
        fn()
    tot = 0.0
    for _ in range(reps):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        tot += a.elapsed_time(b)
    return tot / reps * 1e3   # us


def main():
    M = int(sys.argv[1]) if len(sys.argv) > 1 else 65536
    torch.manual_seed(0)
    x = torch.randn(M, 384, device="cuda").bfloat16()
    w1 = (torch.randn(1536, 384, device="cuda") / math.sqrt(384)).bfloat16()
    w2 = (torch.randn(384, 1536, device="cuda") / math.sqrt(1536)).bfloat16()
    b1, b2 = torch.randn(1536, device="cuda") * 0.1, torch.randn(384, device="cuda") * 0.1
    lw, lb = torch.ones(384, device="cuda"), torch.zeros(384, device="cuda")
    out = torch.empty_like(x)

    def unfused():
        h = L.layernorm(x, lw, lb, 1e-5)
        hid = L.gemm(h, w1, bias=b1, act=L.ACT_GELU)
        L.gemm(hid, w2, bias=b2, residual=x, out=out)

    res = {"M": M, "unfused_us": timed(unfused)}
    res["ff_block_us"] = timed(lambda: L.ff_block(x, lw, lb, w1, b1, w2, b2, out=out))
    flops = 4.0 * M * 384 * 1536
    res["ff_block_tflops"] = flops / (res["ff_block_us"] * 1e-6) / 1e12
    res["unfused_tflops"] = flops / (res["unfused_us"] * 1e-6) / 1e12
    print(json.dumps(res))


if __name__ == "__main__":
    main()
