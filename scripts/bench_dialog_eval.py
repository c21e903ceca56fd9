"""Throughput of the batched VL-LN dialog evaluation loop (HabitatDialogEvaluator.run) for B environments.

    python scripts/bench_dialog_eval.py [--batches 1,8,64] [--episodes 2] [--max-steps 24] [--repeats 3] [--max-new 8]
                                        [--out FILE]

Weights are seeded random at the Qwen2.5-VL-7B shapes, System-2-only (the dialog checkpoint's shape); frames are
480 x 640, resized to 384 x 384 for the history on the device (PIL Qwen2-VL image processor, reproduced by
QwenImagePreprocessor), num_history 8, the instance-dialog prompt with 5 questions per episode.  The environment,
navmesh and follower are the zero-cost stand-ins of bench_habitat_eval.py (the follower walks FORWARD three times per
goal, then STOP); the NPC answers at once with a fixed sentence.  The tokenizer is a word-level stand-in and the random
model's answers are replaced by a scripted cycle per environment -- question, pixel goal, arrows, look-down, question,
pixel goal, arrows -- so two of every seven System-2 turns are questions and each is followed by a dialog turn.

For each B: a warm-up run, then `--repeats` timed runs of `--episodes` episodes per environment with `--max-steps`
steps at most; at B = 8 the same episodes also run one environment at a time (eight B = 1 drivers in turn), alternating
with the batched runs.  Every round is timed on the host with a device synchronise after it.  Reported: environment
steps per second per run and their median, median (min-max) ms per round, System-2 calls, and the rows the dialog turns
prefilled next to the rows a full re-prefill of the same prompts would take.  Card name, power limit and SM clock are
read in the same run.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scripts.bench_habitat_eval import Follower, ScriptedAnswers, SyntheticEnvS2, summary  # noqa: E402
from scripts.bench_realworld_agent import BenchProcessor, card  # noqa: E402

ANSWERS = ["<talk>Is the bed upstairs?", "240, 320", "↑←", "↓", "<talk>Which room is it in?", "200, 300", "→↑"]


class _HabitatEnv:
    def __init__(self, env, sim):
        self.env, self.sim = env, sim

    @property
    def current_episode(self):
        return self.env.get_current_episode()

    @property
    def episode_over(self):
        return self.env.over


class SyntheticDialogEnv(SyntheticEnvS2):
    def __init__(self, *args):
        super().__init__(*args)
        self._env, self.over = _HabitatEnv(self, self._env.sim), False

    def reset(self):
        self.over = False
        return super().reset()

    def step(self, action):
        self.over = int(action) == 0
        return super().step(action)

    def get_current_episode(self):
        ep = super().get_current_episode()
        ep.object_category = "bed"
        ep.instruction.instance_id = ["0"]
        return ep


class Answers(ScriptedAnswers):
    def decode(self, ids, skip_special_tokens=True):
        e = self.order.pop(0)
        n = self.count.get(e, 0)
        self.count[e] = n + 1
        return ANSWERS[n % len(ANSWERS)]


def make_evaluator(model, proc, max_steps, max_new):
    from internnav_b200.habitat_dialog import HabitatDialogEvaluator

    class Timed(HabitatDialogEvaluator):
        def _round(self, req, gens, state, envs):
            s2 = [e for e in sorted(req) if req[e].kind == "s2"]
            proc.tokenizer.order = [self.robots[e] for e in s2]
            self.kinds = [req[e].turn.kind for e in s2]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            super()._round(req, gens, state, envs)
            torch.cuda.synchronize()
            self.round_ms.append((time.perf_counter() - t0) * 1e3)

    ev = Timed(model, proc, task="instance_dialog", turn=5, num_history=8, resize_w=384, resize_h=384,
               max_steps_per_episode=max_steps, max_new_tokens=max_new, camera_height=1.25,
               depth_filter=lambda d, blur_type=None: d, make_follower=Follower,
               npc=lambda qs: ["It is in the bedroom at the end of the corridor."] * len(qs))
    ev.round_ms, ev.kinds = [], []
    return ev


def counted(model, ev):
    """Wrap model.generate: per call, the dialog turns' prefilled rows and prompt lengths go to ev.rows."""
    generate = model.generate

    def gen(prompts, *a, **kw):
        out = generate(prompts, *a, **kw)
        reused = model._s2.last_cache["reused"] if "past_key_values" in kw else [0] * len(prompts)
        for k, p, r in zip(ev.kinds, prompts, reused):
            if k == "dialog":
                ev.rows[0] += len(p) - r
                ev.rows[1] += len(p)
        return out
    model.generate = gen


def run(ev, proc, robots, frames, depth, episodes):
    """Run `episodes` episodes on each listed robot's environment -> (env steps, seconds, round times)."""
    ev.robots, ev.round_ms = robots, []
    proc.tokenizer.count = {}
    envs = [SyntheticDialogEnv(frames[r % len(frames)], depth, r, episodes) for r in robots]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = ev.run(envs)
    torch.cuda.synchronize()
    sec = time.perf_counter() - t0
    assert not any("error" in x for rs in res for x in rs), res
    return sum(e.steps for e in envs), sec, list(ev.round_ms)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,8,64")
    ap.add_argument("--episodes", type=int, default=2)
    ap.add_argument("--max-steps", type=int, default=24)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--max-new", type=int, default=8)
    ap.add_argument("--layers", type=int, default=28)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_dialog_eval needs a GPU")
    from transformers.models.qwen2_vl.image_processing_pil_qwen2_vl import Qwen2VLImageProcessorPil
    from internnav_b200.internvla_n1 import InternVLAN1ForCausalLM
    from oracle import qwen_oracle as Q
    cfg = dict(Q.QWEN25VL_7B, layers=a.layers)
    result = {"card": card(), "cfg": dict(layers=a.layers, max_new_tokens=a.max_new, num_history=8, frame="480x640",
                                          resize="384x384", episodes=a.episodes, max_steps_per_episode=a.max_steps,
                                          repeats=a.repeats, answers=ANSWERS)}
    print(json.dumps(result), flush=True)
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
    for B in [int(x) for x in a.batches.split(",")]:
        robots = list(range(B))
        ev = make_evaluator(model, proc, 6, a.max_new)
        run(ev, proc, robots, frames, depth, 1)                       # warm-up: 6 steps per environment
        ev.max_steps_per_episode = a.max_steps
        one = None
        if B == 8:
            one = make_evaluator(model, proc, 6, a.max_new)
            run(one, proc, [0], frames, depth, 1)
            one.max_steps_per_episode = a.max_steps
        batched, single, s2_calls = [], [], []
        ev.rows = [0, 0]
        counted(model, ev)
        for _ in range(a.repeats):      # batched and one-at-a-time runs alternate
            before = ev.calls["s2"]
            batched.append(run(ev, proc, robots, frames, depth, a.episodes))
            s2_calls.append(ev.calls["s2"] - before)
            print(json.dumps({"B": B, "steps": batched[-1][0], "seconds": round(batched[-1][1], 3)}), flush=True)
            if one is not None:
                del model.generate
                parts = [run(one, proc, [r], frames, depth, a.episodes) for r in robots]
                single.append((sum(p[0] for p in parts), sum(p[1] for p in parts), [m for p in parts for m in p[2]]))
                counted(model, ev)
        del model.generate
        out = {"B": B, "batched": dict(summary(batched), s2_calls=s2_calls,
                                       dialog_rows_prefilled=ev.rows[0], dialog_rows_full_reprefill=ev.rows[1])}
        if single:
            out["one_at_a_time"] = summary(single)
            out["batched_over_one_at_a_time"] = [round((b[0] / b[1]) / (s[0] / s[1]), 2) for b, s in zip(batched, single)]
        result["B%d" % B] = out
        print(json.dumps(out), flush=True)
        del ev, one
        torch.cuda.empty_cache()
    result["card_after"] = card()
    print(json.dumps(result))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()
