"""Served-frame latency of the batched real-world agent (InternVLAN1AsyncAgent.serve) for B robots.

    python scripts/bench_realworld_agent.py [--batches 1,8,64] [--cycles 8] [--max-new 8] [--out FILE]

Weights are seeded random at the Qwen2.5-VL-7B shapes with the nextdit_async System 1; frames are 480 x 640, resized to
384 x 384 for System 2 on the device (the processor's image half is the PIL Qwen2-VL image processor, which
QwenImagePreprocessor reproduces); plan_step_gap = 4 and num_history = 8, so once an episode has 8 frames every fresh
turn carries 9 images.  The tokenizer is a word-level stand-in (no checkpoint files are read), and the random model's
answers are replaced by scripted ones -- a pixel goal, or look-down then a pixel goal -- so that every robot holds a
latent plan; the answers are max_new_tokens long, about the length of a pixel-goal answer.

All robots run in lock step, so every served frame is one of three kinds, told apart by the agent's call counters:
  s1_only   no robot is due: history frames + one System-1 call (generate_traj for B robots, waypoint tail);
  fresh_s2  every robot is due: one System-2 call (9 images per robot) + one System-1 call;
  look_down every robot answers [5]: the fresh call, the look-down call on the same frame, then System 1.
Each frame is timed on the host around `serve` with a device synchronise after it.  After a warm-up episode of 12 frames
(every shape compiled, K/V pool and CUDA graphs built) and 6 look-down frames, `--cycles` cycles of 6 frames (one
System-2 period at plan_step_gap 4) alternate plain and look-down cycles.  Card name, power limit and SM clock are read
in the same run.
"""
import argparse
import json
import os
import re
import statistics
import subprocess
import sys
import time
from types import SimpleNamespace

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


class BenchProcessor:
    """Chat template with Qwen's vision markers, word-level token ids, and scripted answers (see module docstring)."""
    image_token = "<|image_pad|>"
    _SPECIAL = {"<|vision_start|>": 151652, "<|image_pad|>": 151655, "<|vision_end|>": 151653}

    class _Tok:
        padding_side = "left"

        def __init__(self):
            self.mode, self.batch, self.n = "pixel", 1, 0

        def decode(self, ids, skip_special_tokens=True):
            self.n += 1
            if self.mode == "look_down" and ((self.n - 1) // self.batch) % 2 == 0:
                return "↓"
            return "240, 320"

    def __init__(self, image_processor):
        self.image_processor = image_processor
        self.tokenizer = self._Tok()

    def apply_chat_template(self, conversation, tokenize=False, add_generation_prompt=True):
        out = []
        for t in conversation:
            body = "".join("<|vision_start|><|image_pad|><|vision_end|>" if c["type"] == "image" else c["text"]
                           for c in t["content"])
            out.append("<|im_start|>%s\n%s<|im_end|>\n" % (t["role"], body))
        return "".join(out) + ("<|im_start|>assistant\n" if add_generation_prompt else "")

    def __call__(self, text, images=None, return_tensors="pt"):
        assert images is None, "images go through QwenImagePreprocessor"
        ids = []
        for piece in re.split(r"(<\|vision_start\|>|<\|image_pad\|>|<\|vision_end\|>)", text[0]):
            if piece in self._SPECIAL:
                ids.append(self._SPECIAL[piece])
            else:
                ids += [1000 + (sum(map(ord, w)) * 2654435761) % 100000 for w in re.findall(r"\w+|[^\w\s]", piece)]
        return {"input_ids": torch.tensor([ids])}


def run(model, proc, B, cycles, max_new, frames):
    from internnav_b200.agent_realworld import InternVLAN1AsyncAgent
    args = SimpleNamespace(device="cuda:0", model_path=None, resize_w=384, resize_h=384, num_history=8, plan_step_gap=4)
    agent = InternVLAN1AsyncAgent(args, model=model, processor=proc, num_envs=B)
    agent.policy.max_new_tokens = max_new
    assert agent.policy._vl is not None, "System-2 images must take the device path"
    proc.tokenizer.batch = B
    depth = [np.zeros((480, 640), dtype=np.float32)] * B
    ins = ["robot %d: leave the office, pass the red bin and stop at the computer monitor" % b for b in range(B)]
    times = {"s1_only": [], "fresh_s2": [], "look_down": []}
    k = 0

    def serve(timed):
        nonlocal k
        rgbs = list(frames[k % len(frames)][:B])
        before = dict(agent.calls)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = agent.serve(list(range(B)), rgbs, depth, ins, resets=[k == 0] * B)
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1e3
        k += 1
        assert not any(isinstance(r, Exception) for r in res), res
        kind = {(0, 1): "s1_only", (1, 1): "fresh_s2", (2, 1): "look_down"}[
            (agent.calls["s2"] - before["s2"], agent.calls["s1"] - before["s1"])]
        if timed:
            times[kind].append(ms)

    proc.tokenizer.mode, proc.tokenizer.n = "pixel", 0
    for _ in range(12):
        serve(False)
    proc.tokenizer.mode, proc.tokenizer.n = "look_down", 0
    for _ in range(6):                  # warms the look-down shapes
        serve(False)
    for c in range(cycles):
        proc.tokenizer.mode, proc.tokenizer.n = ("pixel", "look_down")[c % 2], 0
        for _ in range(6):
            serve(True)
    out = {"B": B, "frames": k}
    for kind, ms in times.items():
        out[kind] = dict(n=len(ms), ms_median=statistics.median(ms), ms_min=min(ms), ms_max=max(ms)) if ms else None
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,8,64")
    ap.add_argument("--cycles", type=int, default=8)
    ap.add_argument("--max-new", type=int, default=8)
    ap.add_argument("--layers", type=int, default=28)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_realworld_agent needs a GPU")
    from transformers.models.qwen2_vl.image_processing_pil_qwen2_vl import Qwen2VLImageProcessorPil
    from internnav_b200.internvla_n1 import InternVLAN1ForCausalLM
    from internnav_b200.manifest import random_nextdit_state_dict
    from oracle import qwen_oracle as Q
    cfg = dict(Q.QWEN25VL_7B, layers=a.layers)
    result = {"card": card(), "cfg": dict(layers=a.layers, max_new_tokens=a.max_new, plan_step_gap=4, num_history=8,
                                          frame="480x640", resize="384x384")}
    print(json.dumps(result), flush=True)
    model = InternVLAN1ForCausalLM(cfg, device="cuda:0", system1="nextdit_async")
    s2_sd = Q.make_s2_state_dict(cfg, seed=0, device="cuda", dtype=torch.bfloat16, lm_head=True)
    model.load_parts(s2_sd, random_nextdit_state_dict(1, device="cuda", dtype=torch.bfloat16))
    del s2_sd
    torch.cuda.empty_cache()
    proc = BenchProcessor(Qwen2VLImageProcessorPil(min_pixels=3136, max_pixels=12845056))
    batches = [int(x) for x in a.batches.split(",")]
    rng = np.random.default_rng(0)
    frames = [rng.integers(0, 256, (max(batches), 480, 640, 3), dtype=np.uint8) for _ in range(3)]
    for B in batches:
        result["B%d" % B] = run(model, proc, B, a.cycles, a.max_new, frames)
        print(json.dumps(result["B%d" % B]), flush=True)
        torch.cuda.empty_cache()
    result["card_after"] = card()
    print(json.dumps(result))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()
