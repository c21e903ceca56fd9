"""Scenario drivers shared by tests/test_vs_live_reference.py and oracle/gen_golden_live.py.

Each driver runs ONE implementation (the reference's own class, or this project's) through a seeded random scenario and
returns everything the scenario observes as a JSON-able trace.  The scenario's control flow follows the outputs of the
implementation it drives, so two implementations that agree produce the same trace, and the traces recorded from the
reference (tests/golden/live_reference_traces.json) pin this project's classes where the reference is not installed.
"""
import contextlib
import io
import json
from types import SimpleNamespace

import numpy as np
import torch

from oracle import agent_script, policy_script

POLICY_SEEDS = [101, 102, 103]
AGENT_CASES = [(201, "partial_async"), (202, "sync"), (203, "partial_async")]


def _pixel(p):
    return None if p is None else np.asarray(p).tolist()


def policy_trace(seed, reference_net=None):
    """InternVLAN1Net host logic (s2_step / step_no_infer / s1_step_latent / reset).  `reference_net`: the reference's
    InternVLAN1Net class; None drives internnav_b200.policy.InternVLAN1Policy."""
    rng = np.random.Generator(np.random.PCG64(seed))
    answers, trajs = policy_script.random_answers(rng, n=40), policy_script.random_trajs(rng, n=8)
    num_history = int(rng.choice([2, 4, 8]))
    proc = policy_script.FakeProcessor()
    if reference_net is not None:
        net = reference_net(policy_script.ScriptedLLM(answers, trajs), proc, num_history=num_history)
        net.reset()
        s2 = lambda o, look: net.s2_step(o["rgb"], o["depth"], None, o["instruction"], None, look_down=look)
        s1 = lambda: net.s1_step_latent(None, None, torch.zeros(1))
        no_infer = lambda o: net.step_no_infer(o["rgb"], o["depth"], None)
        reset = net.reset
        state = lambda: [net.llm_output, int(net.episode_idx), len(net.rgb_list)]
    else:
        from internnav_b200.policy import InternVLAN1Policy

        class Model:  # the model mirror's two calls, answering from the same script
            def __init__(self):
                self.n, self.nt = 0, 0

            def generate_with_latents(self, prompts, pixel_values, image_grid_thw, max_new_tokens=128):
                ans = answers[self.n % len(answers)]
                self.n += 1
                return SimpleNamespace(generated=[policy_script.encode(ans) + [151645]], latents=torch.zeros(1, 1, 1))

            def generate_traj(self, traj_latents=None, images_dp=None, depths_dp=None):
                t = trajs[self.nt % len(trajs)]
                self.nt += 1
                return torch.tensor(t, dtype=torch.float32)
        net = InternVLAN1Policy(Model(), proc, num_envs=1, num_history=num_history)
        net.reset()
        s2 = lambda o, look: net.s2_step([0], [o["rgb"]], [o["depth"]], [None], [o["instruction"]], None, [look])[0]
        s1 = lambda: net.s1_step_latent([0], [torch.zeros(1, 2, 4, 4, 3)], [torch.zeros(1, 2, 4, 4, 1)], [torch.zeros(1, 1, 1)])[0]
        no_infer = lambda o: net.step_no_infer([0], [o["rgb"]])
        reset = lambda: net.reset([0])
        state = lambda: [net.episodes[0].llm_output, int(net.episodes[0].episode_idx), len(net.episodes[0].rgb_list)]
    trace, look = [], False
    with contextlib.redirect_stdout(io.StringIO()):
        for k in range(45):
            o = agent_script.make_obs(k, size=(24, 32))
            u = rng.random()
            if k == 20:
                reset()
                look = False
            if k == 0 or look or u < 0.5:
                a = s2(o, look)
                action = None if a.output_action is None else [int(x) for x in a.output_action]
                trace.append(["s2", k, proc.log.pop(), state(), _pixel(a.output_pixel), action])
                look = a.output_action is not None and 5 in a.output_action[:1]
                if a.output_latent is not None and rng.random() < 0.6:
                    trace.append(["s1", k, np.asarray(s1().idx).tolist()])
            else:
                no_infer(o)
                trace.append(["noinfer", k])
    return trace


def agent_trace(seed, mode, reference_module_loader=None):
    """InternVLAN1Agent stepped through a scripted policy.  `reference_module_loader`: oracle.ref_loader
    .load_reference_agent (the reference's agent, real S2 worker thread, polling sleeps shortened); None drives
    internnav_b200.agent.InternVLAN1Agent."""
    rng = np.random.Generator(np.random.PCG64(seed))
    script = agent_script.random_script(rng, p_latent=float(rng.uniform(0.3, 0.9)), p_raise=0.05)
    with contextlib.redirect_stdout(io.StringIO()):
        if reference_module_loader is not None:
            holder = {}

            def factory(config=None):
                holder["policy"] = agent_script.ScriptedPolicy(script, s2_output_cls=holder["mod"].S2Output,
                                                               s1_output_cls=holder["mod"].S1Output)
                return holder["policy"]
            mod = holder["mod"] = reference_module_loader(factory)
            settings = dict(policy_name="InternVLAN1_Policy", state_encoder=None, device="cpu", infer_mode=mode,
                            sys2_max_forward_step=8, width=640, height=480, hfov=79, vis_debug=False)
            agent = mod.InternVLAN1Agent(mod.AgentCfg(model_name="internvla_n1", model_settings=settings))
            pol = holder["policy"]
            agent.reset()
            reset = lambda: agent.reset(reset_index=[0])
            state = lambda: [int(agent.dual_forward_step), bool(agent.look_down)]
        else:
            from internnav_b200.agent import InternVLAN1Agent, PerEnvPolicies
            pol = agent_script.ScriptedPolicy(script)
            agent = InternVLAN1Agent(PerEnvPolicies([pol]), num_envs=1, infer_mode=mode, sys2_max_forward_step=8)
            agent.reset()
            reset = lambda: agent.reset([0])
            state = lambda: [int(agent.dual_forward_step[0]), bool(agent.look_down[0])]
        pol.drain()
        trace = []
        for k in range(40):
            if k == 17:
                reset()
            out = agent.step([agent_script.make_obs(k)])
            trace.append([k, json.loads(json.dumps(out[0]["action"], default=lambda x: np.asarray(x).tolist())), pol.drain(), state()])
    return trace
