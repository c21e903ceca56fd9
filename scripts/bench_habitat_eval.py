"""Throughput of the batched VLN-CE evaluation loop (HabitatVLNEvaluator.run_dual_system, or run_system2 with
`--mode system2`) for B environments.

    python scripts/bench_habitat_eval.py [--mode dual_system|system2] [--batches 1,8,64] [--episodes 2] [--max-steps 24]
                                         [--repeats 3] [--max-new 8] [--out FILE]

Weights are seeded random at the Qwen2.5-VL-7B shapes with the nextdit_async System 1 (the released DualVLN head);
frames are 480 x 640, resized to 384 x 384 for System 2 on the device (PIL Qwen2-VL image processor, reproduced by
QwenImagePreprocessor), num_history 8.  The environment is synthetic and costs nothing: it hands out pre-drawn frames
and ends an episode on STOP.  The tokenizer is a word-level stand-in and the random model's answers are replaced by a
scripted cycle per environment -- pixel goal, arrows, look-down, pixel goal, pixel goal, arrows -- as
bench_realworld_agent.py scripts them; System 1's action chunks come from the seeded head.

For each B: a warm-up run (one short episode per environment: every shape compiled, K/V pool and CUDA graphs built),
then `--repeats` timed runs of `--episodes` episodes per environment with `--max-steps` steps at most.  Every round is
timed on the host with a device synchronise after it.  Reported: environment steps per second of each timed run (every
`env.step`, camera moves included) and their median, and the median (min-max) ms per round over all runs.  At B = 8 the
same episodes also run one environment at a time (eight B = 1 drivers in turn), the reference's one-process-per-
environment shape, alternating with the batched runs; the ratio of the two rates is reported per repeat.  Card name,
power limit and SM clock are read in the same run.

`--mode system2` runs the System-2-only model (the same seeded 7B System 2, no System 1) through `run_system2`: the
synthetic environment also carries a zero-cost simulator surface (agent state, a navmesh that accepts every goal) and
the follower answers FORWARD three times per goal, then STOP, so every pixel answer is lifted to a world goal and walked.
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scripts.bench_realworld_agent import BenchProcessor, card  # noqa: E402

ANSWERS = ["240, 320", "↑←", "↓", "200, 300", "260, 330", "→↑"]


class SyntheticEnv:
    """The HabitatEnv surface over pre-drawn frames; counts its steps."""

    def __init__(self, frames, depth, robot, episodes):
        self.frames, self.depth, self.robot, self.n = frames, depth, robot, episodes
        self.is_running, self.i, self.steps, self.k = True, 0, 0, 0

    def _obs(self):
        self.k += 1
        return {"rgb": self.frames[self.k % len(self.frames)], "depth": self.depth, "gps": np.zeros(2)}

    def reset(self):
        if self.i >= self.n:
            self.is_running = False
            return None
        self.i += 1
        return self._obs()

    def step(self, action):
        self.steps += 1
        return self._obs(), 0.0, int(action) == 0, {}

    def get_current_episode(self):
        from types import SimpleNamespace
        return SimpleNamespace(scene_id="data/scene%d/x.glb" % self.robot, episode_id=str(self.i),
                               instruction=SimpleNamespace(instruction_text="robot %d: leave the office, pass the red "
                                                                            "bin and stop at the computer monitor." % self.robot))

    def get_metrics(self):
        return {"success": 0.0, "spl": 0.0, "oracle_success": 0.0, "distance_to_goal": 1.0, "top_down_map": None}


class _Sim:
    """The zero-cost simulator surface of the system2 loop: a fixed agent state and a navmesh that takes every goal."""

    def __init__(self):
        from types import SimpleNamespace
        state = SimpleNamespace(position=np.zeros(3, dtype=np.float32), rotation=SimpleNamespace(w=1.0, x=0.0, y=0.0, z=0.0))
        self.get_agent_state = lambda: state
        self.pathfinder = SimpleNamespace(is_navigable=lambda p: True, snap_point=lambda p: p)


class SyntheticEnvS2(SyntheticEnv):
    def __init__(self, *args):
        super().__init__(*args)
        from types import SimpleNamespace
        self._env = SimpleNamespace(sim=_Sim())

    def _obs(self):
        return dict(super()._obs(), compass=np.zeros(1, dtype=np.float32))


class Follower:
    """FORWARD three times per goal, then STOP."""

    def __init__(self, env):
        self.n = 0

    def get_next_action(self, goal):
        self.n += 1
        return 0 if self.n % 4 == 0 else 1


class ScriptedAnswers(BenchProcessor._Tok):
    """Each environment cycles through ANSWERS; answers are told apart by the order of decode calls within a System-2
    call, which follows the order of the environments the evaluator passes (set by `Timed._round`)."""

    def __init__(self):
        super().__init__()
        self.order, self.count = [], {}

    def decode(self, ids, skip_special_tokens=True):
        e = self.order.pop(0)
        n = self.count.get(e, 0)
        self.count[e] = n + 1
        return ANSWERS[n % len(ANSWERS)]


def make_evaluator(model, proc, max_steps, max_new, mode="dual_system"):
    from internnav_b200.habitat_eval import HabitatVLNEvaluator

    class Timed(HabitatVLNEvaluator):
        def _round(self, req, gens, state):
            proc.tokenizer.order = [self.robots[e] for e in sorted(req) if req[e].kind == "s2"]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            super()._round(req, gens, state)
            torch.cuda.synchronize()
            self.round_ms.append((time.perf_counter() - t0) * 1e3)

    kw = {} if mode == "dual_system" else dict(camera_height=1.25, depth_filter=lambda d, blur_type=None: d,
                                               make_follower=Follower)
    ev = Timed(model, proc, num_history=8, resize_w=384, resize_h=384, max_steps_per_episode=max_steps,
               max_new_tokens=max_new, mode=mode, **kw)
    ev.round_ms = []
    return ev


def run(ev, proc, robots, frames, depth, episodes):
    """Run `episodes` episodes on each listed robot's environment -> (env steps, seconds, round times)."""
    ev.robots, ev.round_ms = robots, []
    proc.tokenizer.count = {}
    system2 = ev.mode == "system2"
    envs = [(SyntheticEnvS2 if system2 else SyntheticEnv)(frames[r % len(frames)], depth, r, episodes) for r in robots]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = ev.run_system2(envs) if system2 else ev.run_dual_system(envs)
    torch.cuda.synchronize()
    sec = time.perf_counter() - t0
    assert not any("error" in x for rs in res for x in rs), res
    return sum(e.steps for e in envs), sec, list(ev.round_ms)


def summary(runs):
    """runs: [(env steps, seconds, round times)] of repeated timed runs -> env steps / s of each run and their median,
    ms per round over all runs."""
    rates = [steps / sec for steps, sec, _ in runs]
    ms = [m for _, _, r in runs for m in r]
    return dict(env_steps=[s for s, _, _ in runs], seconds=[round(sec, 3) for _, sec, _ in runs],
                env_steps_per_s=[round(r, 1) for r in rates], env_steps_per_s_median=round(statistics.median(rates), 1),
                rounds=len(ms), ms_per_round_median=round(statistics.median(ms), 1), ms_per_round_min=round(min(ms), 1),
                ms_per_round_max=round(max(ms), 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", default="dual_system", choices=["dual_system", "system2"])
    ap.add_argument("--batches", default="1,8,64")
    ap.add_argument("--episodes", type=int, default=2)
    ap.add_argument("--max-steps", type=int, default=24)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--max-new", type=int, default=8)
    ap.add_argument("--layers", type=int, default=28)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_habitat_eval needs a GPU")
    from transformers.models.qwen2_vl.image_processing_pil_qwen2_vl import Qwen2VLImageProcessorPil
    from internnav_b200.internvla_n1 import InternVLAN1ForCausalLM
    from internnav_b200.manifest import random_nextdit_state_dict
    from oracle import qwen_oracle as Q
    cfg = dict(Q.QWEN25VL_7B, layers=a.layers)
    result = {"card": card(), "cfg": dict(mode=a.mode, layers=a.layers, max_new_tokens=a.max_new, num_history=8, frame="480x640",
                                          resize="384x384", episodes=a.episodes, max_steps_per_episode=a.max_steps,
                                          repeats=a.repeats)}
    print(json.dumps(result), flush=True)
    system1 = "nextdit_async" if a.mode == "dual_system" else None
    model = InternVLAN1ForCausalLM(cfg, device="cuda:0", system1=system1)
    s2_sd = Q.make_s2_state_dict(cfg, seed=0, device="cuda", dtype=torch.bfloat16, lm_head=True)
    model.load_parts(s2_sd, random_nextdit_state_dict(1, device="cuda", dtype=torch.bfloat16) if system1 else None)
    del s2_sd
    torch.cuda.empty_cache()
    proc = BenchProcessor(Qwen2VLImageProcessorPil(min_pixels=3136, max_pixels=12845056))
    proc.tokenizer = ScriptedAnswers()
    rng = np.random.default_rng(0)
    frames = [[rng.integers(0, 256, (480, 640, 3), dtype=np.uint8) for _ in range(3)] for _ in range(8)]
    depth = np.full((480, 640, 1), 0.3, dtype=np.float32)
    for B in [int(x) for x in a.batches.split(",")]:
        robots = list(range(B))
        ev = make_evaluator(model, proc, 6, a.max_new, a.mode)
        run(ev, proc, robots, frames, depth, 1)                       # warm-up: 6 steps per environment
        ev.max_steps_per_episode = a.max_steps
        one = None
        if B == 8:
            one = make_evaluator(model, proc, 6, a.max_new, a.mode)
            run(one, proc, [0], frames, depth, 1)
            one.max_steps_per_episode = a.max_steps
        batched, single = [], []
        for _ in range(a.repeats):      # batched and one-at-a-time runs alternate
            batched.append(run(ev, proc, robots, frames, depth, a.episodes))
            if one is not None:
                parts = [run(one, proc, [r], frames, depth, a.episodes) for r in robots]
                single.append((sum(p[0] for p in parts), sum(p[1] for p in parts), [m for p in parts for m in p[2]]))
        out = {"B": B, "batched": summary(batched)}
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
