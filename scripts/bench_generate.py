"""Decode-pass timing of n1_llm_generate at the dual-system bench shape (Qwen2.5-VL-7B, random weights, B prompts of
S = 300 tokens incl. one 392x392 image), on a generation plan without a K/V pool and with the image features passed
whole (no row table): wall time of generate(max_new = a) vs generate(max_new = b) -> ms per decode pass, against the
weight-streaming floor (all decoder + lm_head weights once per pass at the measured HBM bandwidth)."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=64)
    ap.add_argument("--short", type=int, default=2)
    ap.add_argument("--long", type=int, default=10)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    from internnav_b200 import _lib
    from internnav_b200.manifest import random_s2_state_dict
    from internnav_b200.qwen import QWEN25VL_7B, System2
    dev = "cuda:0"
    s2 = System2(QWEN25VL_7B, device=dev)
    s2.load_state_dict(random_s2_state_dict(QWEN25VL_7B, seed=0, device=dev, lm_head=True))
    torch.cuda.empty_cache()
    B, grid = args.envs, (1, 28, 28)
    n_tok = 28 * 28 // 4
    rng = np.random.Generator(np.random.PCG64(7))
    prompts = []
    for _ in range(B):
        pre = rng.integers(0, 151643, 12).tolist()
        post = rng.integers(0, 151643, 300 - 14 - n_tok).tolist()
        prompts.append(pre + [151652] + [151655] * n_tok + [151653] + post)
    px = torch.randn(B * 28 * 28, 1176, device=dev).bfloat16()
    grids = [grid] * B
    feats = s2.visual(px, grids)
    res = {}
    for n in (args.short, args.long):
        s2.generate(prompts, None, grids, max_new_tokens=n, eos_token_ids=(), with_latents=True, image_feats=feats)
        torch.cuda.synchronize()
        ts = []
        for _ in range(args.reps):
            _lib.prof_read()
            t0 = time.perf_counter()
            out, lat, passes = s2.generate(prompts, None, grids, max_new_tokens=n, eos_token_ids=(), with_latents=True,
                                           image_feats=feats)
            torch.cuda.synchronize()
            ts.append((time.perf_counter() - t0) * 1e3)
            launches = _lib.prof_read()["total_launches"]
        res[n] = {"ms": min(ts), "passes": passes, "launches": int(launches)}
    per_pass = (res[args.long]["ms"] - res[args.short]["ms"]) / (res[args.long]["passes"] - res[args.short]["passes"])
    c = QWEN25VL_7B
    H, I, L, V = c["hidden"], c["inter"], c["layers"], c["vocab"]
    wbytes = 2 * (L * (H * (H + 2 * c["kv_heads"] * c["head_dim"]) + H * H + 3 * H * I) + V * H)
    peaks = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json"))) \
        if os.path.exists("MEASURED_PEAKS.json") else {}
    print(json.dumps({"envs": B, "prompt_tokens": 300, "generate_ms": {str(k): v for k, v in res.items()},
                      "ms_per_decode_pass": per_pass, "tokens_per_s": B / (per_pass * 1e-3),
                      "weight_bytes_per_pass": wbytes, "achieved_GBps": wbytes / (per_pass * 1e-3) / 1e9,
                      "peaks": peaks}))


if __name__ == "__main__":
    main()
