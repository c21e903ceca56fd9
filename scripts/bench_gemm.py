"""Developer microbenchmark: n1 wgmma GEMM vs cuBLAS (torch.matmul) on the path's shapes.  Prints TFLOP/s."""
import sys

import torch

sys.path.insert(0, ".")
from internnav_b200 import _lib

SHAPES = [  # (M, N, K, act)   act 3 = swiglu
    (19456, 4608, 3584, 0), (19456, 3584, 3584, 0), (19456, 37888, 3584, 3), (19456, 3584, 18944, 0),
    (50176, 3840, 1280, 0), (50176, 1280, 1280, 0), (50176, 6848, 1280, 3), (50176, 1280, 3424, 0),
    (65536, 1152, 384, 0), (65536, 384, 384, 0), (65536, 1536, 384, 1), (65536, 384, 1536, 0),
    (2048, 1152, 384, 0), (2048, 384, 1536, 0), (8192, 8192, 8192, 0),
]


def timeit(fn, iters=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


for M, N, K, act in SHAPES:
    x = torch.randn(M, K, device="cuda").bfloat16()
    w = (torch.randn(N, K, device="cuda") / K ** 0.5).bfloat16()
    out = torch.empty(M, N // 2 if act == 3 else N, device="cuda", dtype=torch.bfloat16)
    t_n1 = timeit(lambda: _lib.gemm(x, w, act=act, out=out))
    t_cb = timeit(lambda: torch.matmul(x, w.t()))
    fl = 2.0 * M * N * K
    print("M=%6d N=%6d K=%6d act=%d  n1 %7.1f us %7.1f TF/s | cublas %7.1f us %7.1f TF/s | ratio %.2f" %
          (M, N, K, act, t_n1 * 1e3, fl / t_n1 / 1e9, t_cb * 1e3, fl / t_cb / 1e9, t_cb / t_n1))

# fused NavDP MLP (384 -> 1536 -> 384 + residual) vs the two-GEMM path
for M in (65536, 2048):
    x = torch.randn(M, 384, device="cuda").bfloat16()
    w1 = (torch.randn(1536, 384, device="cuda") / 384 ** 0.5).bfloat16()
    w2 = (torch.randn(384, 1536, device="cuda") / 1536 ** 0.5).bfloat16()
    b1, b2 = torch.randn(1536, device="cuda"), torch.randn(384, device="cuda")
    res = torch.randn(M, 384, device="cuda").bfloat16()
    hid = torch.empty(M, 1536, device="cuda", dtype=torch.bfloat16)
    out = torch.empty(M, 384, device="cuda", dtype=torch.bfloat16)

    def two():
        _lib.gemm(x, w1, bias=b1, act=1, out=hid)
        _lib.gemm(hid, w2, bias=b2, residual=res, out=out)
    fl = 4.0 * M * 384 * 1536
    for name, fn in (("two GEMMs", two), ("fused cm1", lambda: _lib.fused_mlp(x, w1, b1, w2, b2, residual=res, out=out, cluster=1)),
                     ("fused cm2", lambda: _lib.fused_mlp(x, w1, b1, w2, b2, residual=res, out=out, cluster=2))):
        t = timeit(fn)
        print("MLP M=%6d %-10s %7.1f us %7.1f TF/s" % (M, name, t * 1e3, fl / t / 1e9))
