"""Fresh System-2 calls of an episode with and without the vision-feature pool (ImageFeaturePool).

    python scripts/bench_s2_history.py [--layers 28] [--v-depth 32] [--batches 8,64] [--gap 4] [--warmup 10]
                                       [--repeats 5] [--budget-frames 16] [--out FILE]

Every environment runs an episode of 480 x 640 frames, resized to 384 x 384 on the device as InternVLAN1Policy's device
path does.  Every `--gap` frames there is a fresh System-2 call whose images are the reference's history pick
np.unique(np.linspace(0, t - 1, 8)) and the current frame (9 images at 392 x 392, 196 tokens each, once t >= 8);
QwenImagePreprocessor makes the pixel rows of all environments.  Weights are seeded random at the Qwen2.5-VL-7B shapes,
so the answers are random tokens; max_new_tokens is small so that the vision tower and the prefill dominate.

Three arms: no pool, an unbounded pool (room for every frame of the episode), and the pool InternVLAN1Policy sizes for
`--budget-frames` frames per environment.  The pools are warmed over the first `--warmup` calls of the episode; the
next `--repeats` calls are timed, the arms alternated within each call, and their tokens and latents compared byte for
byte.  The call after that runs once more per arm with the cached workspaces dropped, for the peak memory PyTorch
allocates during a call.  Card name, power limit and SM clock are read in the same run.
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


def history(t, num_history=8):
    return [] if t == 0 else np.unique(np.linspace(0, t - 1, num_history, dtype=np.int32)).tolist()


def episode(s2, cfg, vl, B, gap, warmup, repeats, budget_frames, max_new):
    from internnav_b200.policy import _image_tokens
    from internnav_b200.qwen import ImageFeaturePool
    from oracle import qwen_oracle as Q
    n_calls = warmup + repeats + 1
    t_end = gap * (n_calls - 1)
    rng = np.random.default_rng(B)
    frames = []            # frames[t]: [B, 384, 384, 3] device uint8

    def frames_until(t):
        while len(frames) <= t:
            raw = rng.integers(0, 256, (B, 480, 640, 3), dtype=np.uint8)
            frames.append(vl.resize(raw, (384, 384)))

    frame_rows = _image_tokens(384, 384)
    pools = {
        "unbounded": ImageFeaturePool(s2, B * (t_end + 1) * frame_rows),
        "budget": ImageFeaturePool(s2, B * budget_frames * frame_rows + B * (9 * frame_rows + _image_tokens(480, 640))),
    }
    prng = np.random.Generator(np.random.PCG64(B))

    def inputs(t):
        frames_until(t)
        ids = history(t) + [t]
        px, grids = vl([frames[i][b] for b in range(B) for i in ids])
        grids = grids.tolist()
        n = len(ids)
        prompts = [Q.make_prompt(prng, 60, grids[b * n:(b + 1) * n], 40) for b in range(B)]
        return prompts, px, grids, n

    def call(arm, prompts, px, grids):
        kw = {} if arm == "off" else {"feature_pool": pools[arm]}
        toks, lat, _ = s2.generate(prompts, px, grids, max_new_tokens=max_new, with_latents=True, **kw)
        info = dict(s2.last_features) if arm != "off" else dict(image_hits=0, vit_patches=sum(t * h * w for t, h, w in grids))
        return toks, lat, info

    arms = ("off", "unbounded", "budget")
    for c in range(warmup):
        prompts, px, grids, _ = inputs(c * gap)
        for arm in arms[1:] if c < warmup - 1 else arms:   # the last warm-up call also warms the plain path
            call(arm, prompts, px, grids)
    res = {arm: dict(ms=[], hits=0, images=0, patches=0) for arm in arms}
    same = True
    for c in range(warmup, warmup + repeats):
        prompts, px, grids, _ = inputs(c * gap)
        outs = {}
        order = arms if c % 2 == 0 else arms[::-1]
        for arm in order:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            toks, lat, info = call(arm, prompts, px, grids)
            torch.cuda.synchronize()
            r = res[arm]
            r["ms"].append((time.perf_counter() - t0) * 1e3)
            r["hits"] += info["image_hits"]
            r["images"] += len(grids)
            r["patches"] += info["vit_patches"]
            outs[arm] = (toks, lat.view(torch.int16).cpu())
        for arm in arms[1:]:
            same &= outs[arm][0] == outs["off"][0] and torch.equal(outs[arm][1], outs["off"][1])
    # the next call once more per arm, untimed, with the cached workspaces dropped: peak memory PyTorch allocates during
    # the call (workspaces, pixel rows and call buffers).  The pools are allocated before (pool_gb).
    prompts, px, grids, _ = inputs((warmup + repeats) * gap)
    peak = {}
    for arm in arms:
        s2._ws.clear()
        torch.cuda.empty_cache()
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        call(arm, prompts, px, grids)
        torch.cuda.synchronize()
        peak[arm] = (torch.cuda.max_memory_allocated() - base) / 1e9
    out = dict(B=B, gap=gap, timed_calls=[c * gap for c in range(warmup, warmup + repeats)], bytes_identical=bool(same))
    for arm in arms:
        r = res[arm]
        out[arm] = dict(ms_median=statistics.median(r["ms"]), ms_min=min(r["ms"]), ms_max=max(r["ms"]),
                        image_hit_rate=r["hits"] / r["images"], vit_patches_per_call=r["patches"] / repeats,
                        call_peak_gb=peak[arm])
        if arm != "off":
            out[arm]["pool_gb"] = pools[arm].bytes / 1e9
            out[arm]["pool_rows"] = pools[arm].rows
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=28)
    ap.add_argument("--v-depth", type=int, default=32)
    ap.add_argument("--batches", default="8,64")
    ap.add_argument("--gap", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--budget-frames", type=int, default=16)
    ap.add_argument("--max-new", type=int, default=8)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_s2_history needs a GPU")
    from transformers.models.qwen2_vl.image_processing_pil_qwen2_vl import Qwen2VLImageProcessorPil
    from internnav_b200.preprocess import QwenImagePreprocessor
    from internnav_b200.qwen import System2
    from oracle import qwen_oracle as Q
    vl = QwenImagePreprocessor.from_hf(Qwen2VLImageProcessorPil(min_pixels=3136, max_pixels=12845056), "cuda:0")
    assert vl is not None
    cfg = dict(Q.QWEN25VL_7B)
    full_att = [i for i in cfg["fullatt"] if i < a.v_depth] or [a.v_depth - 1]
    cfg.update(layers=a.layers, v_depth=a.v_depth, fullatt=full_att)
    result = {"card": card(), "cfg": dict(layers=a.layers, v_depth=a.v_depth, max_new_tokens=a.max_new,
                                          budget_frames=a.budget_frames)}
    print(json.dumps(result), flush=True)
    sd = Q.make_s2_state_dict(cfg, seed=0, device="cuda", dtype=torch.bfloat16, lm_head=True)
    s2 = System2(cfg, device="cuda:0")
    s2.load_state_dict(sd)
    del sd
    torch.cuda.empty_cache()
    for B in (int(x) for x in a.batches.split(",")):
        result["B%d" % B] = episode(s2, cfg, vl, B, a.gap, a.warmup, a.repeats, a.budget_frames, a.max_new)
        print(json.dumps(result["B%d" % B]), flush=True)
    result["card_after"] = card()
    print(json.dumps(result))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()
