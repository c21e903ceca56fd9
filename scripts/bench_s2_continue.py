"""Look-down turn of System 2: full re-prefill against continuing the conversation on its K/V cache.

    python scripts/bench_s2_continue.py [--layers 28] [--v-depth 32] [--batches 8,64] [--repeats 7] [--out FILE]

Turn 1 of every environment holds 9 images at 392 x 392 (8 history frames + the current one, 196 tokens each); turn 2
adds the assistant's answer and a user turn with a 640 x 480 look-down frame (grid 34 x 46, 391 tokens).  Weights are
seeded random at the Qwen2.5-VL-7B shapes, so the answers are random tokens; max_new_tokens is small so that the prefill
dominates.  Both forms run alternated, `--repeats` times each, in one process.  Then the attention alone on the
suffix shape at B = 64: the chunk kernel (attention_cache_wgmma.cu) against the mma.sync kernel (attention.cu), CUDA
events around each launch with the L2 flushed before it, and the image digest pass alone.  Card name, power limit and SM
clock are read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def whole_call(s2, cfg, B, repeats, max_new):
    from internnav_b200.qwen import KVCache, KVPool
    from oracle import qwen_oracle as Q
    rng = np.random.Generator(np.random.PCG64(B))
    g1, gl = [(1, 28, 28)] * 9, (1, 34, 46)
    p1 = [Q.make_prompt(rng, 60, g1, 40) for _ in range(B)]
    npx1 = sum(t * h * w for t, h, w in g1)
    px1 = torch.randn(B * npx1, 1176, device="cuda").bfloat16()
    pool = KVPool(s2, B, 9 * 196 + 391 + 2 * max_new + 512 + cfg["n_query"])
    toks1, _, _ = s2.generate(p1, px1, g1 * B, max_new_tokens=max_new, with_latents=True,
                              past_key_values=[pool.handle(b) for b in range(B)])
    prev = s2.last_cache["caches"]
    p2 = [p + t + Q.make_prompt(rng, 6, [gl], 5) for p, t in zip(p1, toks1)]
    pxl = torch.randn(B, gl[1] * gl[2], 1176, device="cuda").bfloat16()
    px2 = torch.cat([torch.cat([px1[b * npx1:(b + 1) * npx1], pxl[b]]) for b in range(B)])
    g2 = (g1 + [gl]) * B
    res = {"full": [], "cont": []}

    def call(form):
        if form == "full":
            s2.generate(p2, px2, g2, max_new_tokens=max_new, with_latents=True)
        else:
            s2.generate(p2, px2, g2, max_new_tokens=max_new, with_latents=True,
                        past_key_values=[KVCache(pool, h.slot, h.tokens, h.images) for h in prev])
    for _ in range(repeats):
        for form in ("full", "cont"):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            call(form)
            torch.cuda.synchronize()
            res[form].append((time.perf_counter() - t0) * 1e3)
    # peak device memory of one call of each form, untimed: what PyTorch allocates during the call (the workspaces,
    # image features and call buffers) with the cached workspaces dropped first.  The packed weights and the pool are
    # the library's own allocations, shared by both forms (pool_gb below).
    info = {}
    for form in ("full", "cont"):
        s2._ws.clear()
        torch.cuda.empty_cache()
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        call(form)
        torch.cuda.synchronize()
        info[form] = dict(call_peak_gb=(torch.cuda.max_memory_allocated() - base) / 1e9)
    c = s2.last_cache
    # the continuation's image digest pass alone (every image's uploaded rows), CUDA events, median of `repeats`
    dts = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        s2.image_digests(px2, g2)
        b.record()
        torch.cuda.synchronize()
        dts.append(a.elapsed_time(b))
    n_patches = B * (9 * 784 + gl[1] * gl[2])
    out = {}
    for form in ("full", "cont"):
        ms = res[form]
        out[form] = dict(ms_median=statistics.median(ms), ms_min=min(ms), ms_max=max(ms),
                         prefill_rows=sum(len(p) for p in p2) if form == "full" else c["prefill_rows"],
                         vit_patches=n_patches if form == "full" else c["vit_patches"], **info[form])
    out["digest_ms"] = dict(median=statistics.median(dts), min=min(dts), max=max(dts), images=len(g2))
    out["pool_gb"] = pool.bytes / 1e9
    out["reused_rows_mean"] = float(np.mean(c["reused"]))
    return out


def attention_alone(B, ctx, n, iters=20):
    from internnav_b200 import _lib
    hq, hk, hd = 28, 4, 128
    Lk = ctx + n
    qkv = torch.randn(B * n, (hq + 2 * hk) * hd, device="cuda").bfloat16()
    q = qkv[:, :hq * hd]
    K = torch.randn(B * Lk, hk * hd, device="cuda").bfloat16()
    V = torch.randn(B * Lk, hk * hd, device="cuda").bfloat16()
    cu_q = torch.arange(0, B + 1, dtype=torch.int32, device="cuda") * n
    cu_k = torch.arange(0, B + 1, dtype=torch.int32, device="cuda") * Lk
    ctx_t = torch.full((B,), ctx, dtype=torch.int32, device="cuda")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    runs = {
        "wgmma_chunk": lambda: _lib.attention_cache(q, K, V, hq, hk, cu_q, ctx_t, cu_k[:-1].contiguous(), n),
        "mma_sync": lambda: _lib.attention(q, K, V, hq, hk, hd, B, 0, 0, cu_q=cu_q, cu_k=cu_k, max_seq_q=n, causal=True),
    }
    outs = {k: f() for k, f in runs.items()}
    flops = 4.0 * hd * hq * B * sum(ctx + i + 1 for i in range(n))
    res = {"rel_diff": ((outs["wgmma_chunk"].float() - outs["mma_sync"].float()).norm() /
                        outs["mma_sync"].float().norm()).item(), "B": B, "ctx": ctx, "suffix": n}
    for k, f in runs.items():
        ts = []
        for _ in range(iters):
            flush.zero_()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            f()
            b.record()
            torch.cuda.synchronize()
            ts.append(a.elapsed_time(b))
        ms = statistics.median(ts)
        res[k] = dict(ms_median=ms, ms_min=min(ts), ms_max=max(ts), tflops=flops / ms / 1e9)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=28)
    ap.add_argument("--v-depth", type=int, default=32)
    ap.add_argument("--batches", default="8,64")
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--max-new", type=int, default=8)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_s2_continue needs a GPU")
    from internnav_b200.qwen import System2
    from oracle import qwen_oracle as Q
    cfg = dict(Q.QWEN25VL_7B)
    full_att = [i for i in cfg["fullatt"] if i < a.v_depth] or [a.v_depth - 1]
    cfg.update(layers=a.layers, v_depth=a.v_depth, fullatt=full_att)
    result = {"card": card(), "cfg": dict(layers=a.layers, v_depth=a.v_depth, max_new_tokens=a.max_new)}
    result["attention_B64"] = attention_alone(64, 9 * 196 + 9 * 2 + 100 + a.max_new + 6, 391 + 2 + 11)
    print(json.dumps(result["attention_B64"]), flush=True)
    sd = Q.make_s2_state_dict(cfg, seed=0, device="cuda", dtype=torch.bfloat16, lm_head=True)
    s2 = System2(cfg, device="cuda:0")
    s2.load_state_dict(sd)
    del sd
    torch.cuda.empty_cache()
    for B in (int(x) for x in a.batches.split(",")):
        result["B%d" % B] = whole_call(s2, cfg, B, a.repeats, a.max_new)
        print(B, json.dumps(result["B%d" % B]), flush=True)
    result["card_after"] = card()
    print(json.dumps(result))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()
