"""Slotted against paged K/V pools: the attention kernels that read the pool, and the batched dialog loop.

    python scripts/bench_kv_pages.py [--iters 50] [--rounds 5] [--dialog-repeats 3] [--b64-tokens-per-env 0] [--out FILE]

Kernels (CUDA events, `--iters` launches per sample, layouts alternated over `--rounds` rounds, 7B shapes: 28 query /
4 K-V heads, head_dim 128): the decode pass (1 row per sequence) and the latent pass (5 rows) on attn_kernel, and a
200-row continuation chunk on attn_cache_kernel, at B = 8 and 64 with contexts drawn from 2 000 - 3 000 keys.  Three
layouts of the same keys: the slotted pool (sequence b at b * capacity), pages in order, pages shuffled.

Dialog loop (the setting of scripts/bench_dialog_eval.py: seeded 7B System-2-only weights, 480 x 640 frames, 384 x 384
history, num_history 8, scripted answers with two questions in seven turns): B = 8 with the slotted pool and with a paged
pool of the same total tokens, alternated, reporting env steps / s, pages held after each round (median, max) and pool
bytes; then B = 64 on a paged budget (`--b64-tokens-per-env`, default: the B = 8 run's largest per-environment holding
plus one conversation's bound), reporting env steps / s, the pool, the System-2 workspaces and device memory, or where
the memory went if it does not fit.  Card name, power limit and SM clock are read in the same run.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scripts.bench_dialog_eval import ANSWERS, Answers, make_evaluator, run  # noqa: E402
from scripts.bench_realworld_agent import BenchProcessor, card  # noqa: E402

PAGE, HQ, HKV, HD = 64, 28, 4, 128


def _med(xs):
    return round(float(np.median(xs)), 4)


def kernels(iters, rounds):
    from internnav_b200 import _lib
    out = {}
    gen = torch.Generator().manual_seed(0)
    for B in (8, 64):
        klen = torch.randint(2000, 3001, (B,), generator=gen)
        per = -(-3000 // PAGE) - (-205 // PAGE)   # context + a 200-row chunk
        cap = per * PAGE
        n_pages = B * per
        kv = lambda rows: torch.randn(rows, HKV * HD, generator=gen).to(torch.bfloat16).cuda()
        k_s, v_s = kv(B * cap), kv(B * cap)
        # the same keys on pages: in order, and shuffled
        layouts = {"slotted": (k_s, v_s, None)}
        for name, order in (("pages_in_order", torch.arange(n_pages)), ("pages_shuffled", torch.randperm(n_pages, generator=gen))):
            table = order.view(B, per).to(torch.int32)
            k_p = torch.empty_like(k_s)
            v_p = torch.empty_like(v_s)
            dst = (table.long()[:, :, None] * PAGE + torch.arange(PAGE)[None, None, :]).reshape(-1).cuda()
            k_p[dst], v_p[dst] = k_s, v_s
            layouts[name] = (k_p, v_p, table.flatten().cuda())
        row0 = torch.arange(B, dtype=torch.int32, device="cuda") * cap
        res = {}
        for kind, sq in (("decode", 1), ("latent", 5), ("continuation", 200)):
            q = torch.randn(B * sq, HQ * HD, generator=gen).to(torch.bfloat16).cuda()
            o = torch.empty(B * sq, HQ * HD, dtype=torch.bfloat16, device="cuda")
            kl = (klen + (sq if kind != "continuation" else 200)).to(torch.int32).cuda()
            if kind == "continuation":
                cu = torch.arange(B + 1, dtype=torch.int32, device="cuda") * sq
                ctx = klen.to(torch.int32).cuda()

            def launch(name):
                k, v, pages = layouts[name]
                if kind == "continuation":
                    _lib.attention_cache(q, k, v, HQ, HKV, cu, ctx, row0, sq, out=o, pages=pages)
                elif pages is None:
                    _lib.attention_test(q, k, v, o, HQ, HKV, HD, B, seq_q=sq, causal=True, k_len=kl, k_slot=cap)
                else:
                    _lib.attention_paged_test(q, k, v, o, HQ, HKV, B, sq, kl, row0, pages)
            outs = {}
            for name in layouts:   # warm-up and outputs
                launch(name)
                torch.cuda.synchronize()
                outs[name] = o.clone()
            same = all(torch.equal(outs[n].view(torch.int16), outs["slotted"].view(torch.int16)) for n in outs)
            times = {n: [] for n in layouts}
            for _ in range(rounds):
                for name in layouts:
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record()
                    for _ in range(iters):
                        launch(name)
                    b.record()
                    b.synchronize()
                    times[name].append(a.elapsed_time(b) * 1e3 / iters)
            res[kind] = dict(bit_equal=same, **{n: dict(median_us=_med(t), min_us=_med(min(t)), max_us=_med(max(t)))
                                                for n, t in times.items()})
            print(json.dumps({"B": B, kind: res[kind]}), flush=True)
        out["B%d" % B] = dict(context_keys=[int(klen.min()), int(klen.max())], **res)
    return out


def _pool_watch(ev, held):
    """Record the pages the paged pool holds after every round."""
    inner = ev._round

    def rnd(*a, **kw):
        r = inner(*a, **kw)
        pool = ev.policy._kv_pool
        if pool is not None and pool.paged:
            held.append(pool.pages - pool.free_pages)
        return r
    ev._round = rnd


def _ws_bytes(model):
    return {str(k[0]): int(v.numel()) for k, v in model._s2._ws.items()}


def dialog(model, proc, frames, depth, repeats, b64_tokens, b64_only=False):
    out = {}
    if b64_only:
        return dict(B64=b64(model, proc, frames, depth, b64_tokens))
    # ---- B = 8: slotted against paged of the same total tokens
    B, robots = 8, list(range(8))
    evs = {}
    for kind in ("slotted", "paged"):
        ev = make_evaluator(model, proc, 6, 8)
        if kind == "paged":
            cap = evs["slotted"].policy._kv_capacity(480, 640)
            ev.kv_pool_tokens = B * cap
        run(ev, proc, robots, frames, depth, 1)   # warm-up, makes the pools
        ev.max_steps_per_episode = 24
        ev.held = []
        _pool_watch(ev, ev.held)
        evs[kind] = ev
    runs = {k: [] for k in evs}
    for _ in range(repeats):
        for kind, ev in evs.items():
            ev.held.clear()
            steps, sec, _ = run(ev, proc, robots, frames, depth, 2)
            runs[kind].append(dict(steps=steps, seconds=round(sec, 3), held=list(ev.held)))
            print(json.dumps({"B": 8, "pool": kind, "steps": steps, "seconds": round(sec, 3)}), flush=True)
    b8 = {}
    for kind, ev in evs.items():
        r = runs[kind]
        d = dict(env_steps_per_s=[round(x["steps"] / x["seconds"], 2) for x in r], pool_bytes=ev.policy._kv_pool.bytes,
                 slot_tokens=ev.policy._kv_capacity(480, 640))
        d["median_env_steps_per_s"] = _med(d["env_steps_per_s"])
        if kind == "paged":
            held = [h for x in r for h in x["held"]]
            d.update(pool_pages=ev.policy._kv_pool.pages, pages_held_median=_med(held), pages_held_max=int(max(held)),
                     evictions=ev.policy._kv_pool.evictions)
        b8[kind] = d
    out["B8"] = b8
    print(json.dumps({"B8": b8}), flush=True)
    max_held = b8["paged"]["pages_held_max"]
    slot_tokens = b8["paged"]["slot_tokens"]
    del evs
    out["B64"] = b64(model, proc, frames, depth, b64_tokens or (-(-max_held // 8) * PAGE + slot_tokens))
    return out


def b64(model, proc, frames, depth, per_env):
    """B = 64 on a paged budget of per_env tokens per environment."""
    model._s2._ws.clear()
    torch.cuda.empty_cache()
    budget = 64 * per_env
    free0, total = torch.cuda.mem_get_info()
    torch.cuda.reset_peak_memory_stats()
    ev = make_evaluator(model, proc, 6, 8)
    ev.kv_pool_tokens = budget
    ev.held = []
    _pool_watch(ev, ev.held)
    r = dict(kv_pool_tokens=budget, tokens_per_env=per_env, device_free_before_bytes=int(free0),
               device_total_bytes=int(total))
    try:
        run(ev, proc, list(range(64)), frames, depth, 1)   # warm-up
        ev.max_steps_per_episode = 24
        ev.held.clear()
        steps, sec, _ = run(ev, proc, list(range(64)), frames, depth, 1)
        r.update(fits=True, steps=steps, seconds=round(sec, 3), env_steps_per_s=round(steps / sec, 2),
                   pages_held_median=_med(ev.held), pages_held_max=int(max(ev.held)), evictions=ev.policy._kv_pool.evictions)
    except (torch.cuda.OutOfMemoryError, RuntimeError) as e:
        r.update(fits=False, error=str(e)[:300])
    pool = ev.policy._kv_pool if ev.policy is not None else None
    fp = ev.policy._feature_pool if ev.policy is not None else None
    free1, _ = torch.cuda.mem_get_info()
    r.update(pool_bytes=None if pool is None else pool.bytes, feature_pool_bytes=None if fp is None else fp.bytes,
               s2_workspace_bytes=_ws_bytes(model), torch_max_memory_allocated=int(torch.cuda.max_memory_allocated()),
               torch_memory_reserved=int(torch.cuda.memory_reserved()), device_used_after_bytes=int(total - free1))
    print(json.dumps({"B64": r}), flush=True)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--dialog-repeats", type=int, default=3)
    ap.add_argument("--b64-tokens-per-env", type=int, default=0)
    ap.add_argument("--skip-dialog", action="store_true")
    ap.add_argument("--skip-kernels", action="store_true")
    ap.add_argument("--b64-only", action="store_true", help="skip the B = 8 comparison (needs --b64-tokens-per-env)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_kv_pages needs a GPU")
    result = {"card": card(), "cfg": dict(iters=a.iters, rounds=a.rounds, dialog_repeats=a.dialog_repeats,
                                          answers=ANSWERS)}
    print(json.dumps(result), flush=True)
    if not a.skip_kernels:
        result["kernels"] = kernels(a.iters, a.rounds)
    if not a.skip_dialog:
        from transformers.models.qwen2_vl.image_processing_pil_qwen2_vl import Qwen2VLImageProcessorPil
        from internnav_b200.internvla_n1 import InternVLAN1ForCausalLM
        from oracle import qwen_oracle as Q
        cfg = dict(Q.QWEN25VL_7B)
        model = InternVLAN1ForCausalLM(cfg, device="cuda:0", system1=None)
        s2_sd = Q.make_s2_state_dict(cfg, seed=0, device="cuda", dtype=torch.bfloat16, lm_head=True)
        model.load_parts(s2_sd, None)
        del s2_sd
        torch.cuda.empty_cache()
        proc = BenchProcessor(Qwen2VLImageProcessorPil(min_pixels=3136, max_pixels=12845056))
        proc.tokenizer = Answers()
        rng = np.random.default_rng(0)
        frames = [[rng.integers(0, 256, (480, 640, 3), dtype=np.uint8) for _ in range(3)] for _ in range(8)]
        depth = np.full((480, 640, 1), 0.3, dtype=np.float32)
        result["dialog"] = dialog(model, proc, frames, depth, a.dialog_repeats, a.b64_tokens_per_env, a.b64_only)
    result["card_after"] = card()
    print(json.dumps(result))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()
