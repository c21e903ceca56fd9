"""Decoder-prefill attention at the benchmark shape (64 sequences x 304 tokens, 28 / 4 heads, head_dim 128, causal):
wgmma kernel (attention_wgmma.cu) vs the mma.sync kernel it replaces, CUDA events, L2 flushed.  One JSON line."""
import json
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
    return tot / reps * 1e3


B, S, Hq, Hkv, hd = 64, 304, 28, 4, 128
qkv = torch.randn(B * S, (Hq + 2 * Hkv) * hd, device="cuda").bfloat16()
q, k, v = qkv[:, :Hq * hd], qkv[:, Hq * hd:(Hq + Hkv) * hd], qkv[:, (Hq + Hkv) * hd:]
cu = torch.arange(0, (B + 1) * S, S, dtype=torch.int32, device="cuda")
t_tc = timed(lambda: L.attention_varlen(q, k, v, Hq, Hkv, hd, cu, S, causal=True))
t_old = timed(lambda: L.attention(q, k, v, Hq, Hkv, hd, B, 0, 0, cu_q=cu, cu_k=cu, max_seq_q=S, causal=True))
flops = 4.0 * B * Hq * S * S * hd / 2
print(json.dumps({"shape": "64 x 304 tokens, 28/4 heads, hd 128, causal", "wgmma_us": t_tc, "mma_sync_us": t_old,
                  "speedup": t_old / t_tc, "wgmma_tflops": flops / (t_tc * 1e-6) / 1e12,
                  "causal_gflop": flops / 1e9}))
