"""The two configurations without an asynchronous System 1 against their asynchronous counterparts, at 64 environments
with Qwen2.5-VL-7B / DiT shapes and seeded weights:

  1. trajectories: the synchronous NextDiT head's generate_traj (4 condition tokens, no RGB branch) against the
     asynchronous head's (36 tokens: DINOv2 + MemoryEncoder + QFormer), 32 trajectories per environment, guidance 1.0;
  2. System 2 of a fresh policy turn: the System-2-only model's generate (what s2_step calls for it) against the dual
     model's generate_with_latents (the same decode plus the TRAJ pass), one 392 x 392 image and 104 text tokens per
     prompt, max_new_tokens 32 (seeded weights rarely emit an eos id, so every call decodes the whole budget).

The two arms of a pair alternate, 7 timed calls each after a warm-up, CUDA events around whole calls.  The card's name and
power limit are read in the same run.  Prints one JSON line.  Usage: python scripts/bench_system1_configs.py"""
import json
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, ".")
from internnav_b200.internvla_n1 import InternVLAN1ForCausalLM  # noqa: E402
from internnav_b200.manifest import random_nextdit_state_dict, random_s2_state_dict  # noqa: E402
from internnav_b200.nextdit import NextDiTSystem1  # noqa: E402
from internnav_b200.qwen import QWEN25VL_7B  # noqa: E402
from oracle import qwen_oracle as Q  # noqa: E402

B, NS, CALLS, MAX_NEW = 64, 32, 7, 32


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def _alternate(arms):
    """{name: fn} -> {name: [ms of each call]}: one warm-up call each, then CALLS rounds in alternation."""
    for fn in arms.values():
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(CALLS):
        for k, fn in arms.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            torch.cuda.synchronize()
            times[k].append(a.elapsed_time(b))
    return times


def _summary(times):
    return {k: {"median_ms": float(np.median(v)), "min_ms": float(np.min(v)), "max_ms": float(np.max(v))}
            for k, v in times.items()}


def main():
    torch.backends.cuda.matmul.allow_tf32 = False
    out = {"card": _card(), "environments": B}
    # 1. trajectory heads
    g = torch.Generator().manual_seed(0)
    lat = torch.randn(B, 4, 3584, generator=g).bfloat16().cuda()
    img = torch.rand(B, 2, 224, 224, 3, generator=g).cuda()
    x0 = torch.randn(B * NS, 32, 3, generator=g).bfloat16().cuda()
    heads = {name: NextDiTSystem1(asynchronous=a).load_state_dict(random_nextdit_state_dict(0, asynchronous=a))
             for name, a in (("nextdit", False), ("nextdit_async", True))}
    t = _alternate({name: (lambda h=h: h.generate_traj(lat, img, num_sample_trajs=NS, x_init=x0)) for name, h in heads.items()})
    out["generate_traj"] = dict(_summary(t), trajectories_per_env=NS)
    del heads
    torch.cuda.empty_cache()
    # 2. System 2 of a fresh turn
    sd = random_s2_state_dict(QWEN25VL_7B, seed=0, lm_head=True)
    s2only = InternVLAN1ForCausalLM(system1=None)
    s2only.load_state_dict({k: v for k, v in sd.items() if k != "model.latent_queries"})
    dual = InternVLAN1ForCausalLM(system1="nextdit")     # its System 1 is not called here
    dual._s2.load_state_dict(sd)
    del sd
    torch.cuda.empty_cache()
    rng = np.random.Generator(np.random.PCG64(1))
    grids = [(1, 28, 28)] * B
    prompts = [Q.make_prompt(rng, 80, [grid], 24) for grid in grids]
    px = torch.randn(B * 784, 1176, generator=torch.Generator().manual_seed(2)).bfloat16().cuda()
    t = _alternate({"system2_only_generate": lambda: s2only.generate(prompts, px, grids, max_new_tokens=MAX_NEW),
                    "dual_generate_with_latents": lambda: dual.generate_with_latents(prompts, px, grids,
                                                                                     max_new_tokens=MAX_NEW)})
    a = s2only.generate(prompts, px, grids, max_new_tokens=MAX_NEW, return_dict_in_generate=True).generated
    b = dual.generate_with_latents(prompts, px, grids, max_new_tokens=MAX_NEW).generated
    out["s2_fresh_turn"] = dict(_summary(t), max_new_tokens=MAX_NEW, same_tokens=a == b)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
