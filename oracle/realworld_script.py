"""Scripted processor and models for the real-world agent (InternVLAN1AsyncAgent) -- TEST INFRASTRUCTURE.

Drives the reference class (oracle/gen_golden_realworld.py) and the batched agent of internnav_b200/agent_realworld.py
(tests/test_realworld_agent_*.py) with the same scripted System 2 and System 1, and logs every model call:

  ScriptedProcessor        chat template as plain text with <image> placeholders; `__call__` "tokenises" every character
                           as 1000 + ord and logs the chat text and a digest of every attached image;
  ScriptedReferenceModel   `generate` / `generate_latents` / `generate_traj` of the reference model (one robot);
  ScriptedBatchedModel     `generate_with_latents` / `generate_traj` of the n1b200 model mirror (any number of robots).

Each prompt names its robot ("robot <r>: ..." in the instruction); robot r answers with answers[r][n] on its n-th
System-2 call and its latent plan is the tag 1000 r + n.  `generate_traj` returns trajectories that are a function of
the tag and of a digest of the uint8 System-1 frames it is given (recovered as round(x * 255)), so a wrong frame pairing,
goal frame or resize changes the output.
"""
import hashlib
import re
from types import SimpleNamespace

import numpy as np
import torch

CHAR0, EOS = 1000, 151645
NS, T = 4, 8                       # trajectories per robot and steps per trajectory of the scripted System 1
HEIGHT, WIDTH = 480, 640
_ROBOT_RE = re.compile(r"robot (\d+):")


def instruction(robot):
    return "robot %d: leave the office, pass the red bin and stop at the computer monitor" % robot


def frame(seed, k):
    """Frame k of episode `seed`: rgb uint8 [480, 640, 3] and depth float32 [480, 640] (metres)."""
    rng = np.random.Generator(np.random.PCG64([seed, k]))
    rgb = rng.integers(0, 256, size=(HEIGHT, WIDTH, 3), dtype=np.uint8)
    depth = rng.uniform(0.1, 6.0, size=(HEIGHT, WIDTH)).astype(np.float32)
    return rgb, depth


def digest(a):
    a = np.ascontiguousarray(np.asarray(a))
    return hashlib.sha1(repr((a.shape, str(a.dtype))).encode() + a.tobytes()).hexdigest()[:16]


def s1_digest(images_dp):
    """Digest of the uint8 bytes behind System-1 frames given as x / 255 ([..., 2, 224, 224, 3], any float dtype)."""
    x = torch.as_tensor(images_dp).detach().cpu().double().numpy()
    return digest(np.rint(x * 255.0).astype(np.uint8))


def random_answers(rng, n=40, p_error=0.0):
    """Pixel goals, arrow runs, STOP, an answer without any action (-> []), look-down, and (p_error) a lone number,
    which the reference's pixel parsing cannot read (IndexError)."""
    out = []
    for _ in range(n):
        u = rng.random()
        if u < p_error:
            out.append("%d" % int(rng.integers(0, 480)))
        elif u < p_error + 0.45:
            y, x = int(rng.integers(0, HEIGHT)), int(rng.integers(0, WIDTH))
            out.append(str(rng.choice(["%d, %d", "(%d, %d)", "The next waypoint is at %d %d."])) % (y, x))
        elif u < p_error + 0.62:
            out.append("↓")
        elif u < p_error + 0.7:
            out.append("STOP")
        elif u < p_error + 0.76:
            out.append("I cannot tell where to go.")
        else:
            out.append("".join(rng.choice(["↑", "←", "→"], size=int(rng.integers(1, 5)))))
    return out


def trajectory(tag, frames_digest):
    """Scripted System-1 output of one robot: fp32 [NS, T, 3] deltas from the latent tag and the frames' digest."""
    seed = int(hashlib.sha1(("%d:%s" % (tag, frames_digest)).encode()).hexdigest()[:12], 16)
    rng = np.random.Generator(np.random.PCG64(seed))
    fwd = rng.uniform(0.0, 1.2, size=(NS, T, 1))
    lat = rng.normal(0.0, 0.4, size=(NS, T, 1))
    yaw = rng.normal(0.0, 0.1, size=(NS, T, 1))
    return torch.from_numpy(np.concatenate([fwd, lat, yaw], axis=-1).astype(np.float32))


class _Batch(dict):
    """BatchFeature stand-in: mapping (for **inputs) with attribute access and .to()."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e

    def to(self, device):
        return self


class _Tokenizer:
    padding_side = "left"

    def decode(self, ids, skip_special_tokens=True):
        return "".join(chr(int(i) - CHAR0) for i in ids if CHAR0 <= int(i) < 151643)


class ScriptedProcessor:
    def __init__(self, log):
        self.tokenizer = _Tokenizer()
        self.log = log

    def apply_chat_template(self, conversation, tokenize=False, add_generation_prompt=True):
        out = ["<|%s|>%s" % (t["role"], "".join("<image>" if c["type"] == "image" else c["text"] for c in t["content"]))
               for t in conversation]
        return "\n".join(out) + ("\n<|assistant|>" if add_generation_prompt else "")

    def __call__(self, text, images=None, return_tensors="pt"):
        assert len(text) == 1
        images = images or []
        pieces = text[0].split("<image>")
        assert len(pieces) == len(images) + 1, "placeholders and images do not match"
        ids = []
        for i, piece in enumerate(pieces):
            ids += [CHAR0 + ord(c) for c in piece]
            if i < len(images):
                ids += [151652, 151655, 151653]
        self.log.append({"s2": text[0], "images": [digest(np.asarray(im)) for im in images]})
        n = max(len(images), 1)
        return _Batch(input_ids=torch.tensor([ids]), pixel_values=torch.zeros(4 * n, 4),
                      image_grid_thw=torch.tensor([[1, 2, 2]] * len(images), dtype=torch.int64).reshape(-1, 3))


class _Answers:
    """Per-robot answer scripts and call counters (shared by both model stand-ins)."""

    def __init__(self, answers):
        self.answers = {int(r): list(a) for r, a in answers.items()}
        self.count = {r: 0 for r in self.answers}

    def next(self, prompt_ids):
        text = "".join(chr(int(i) - CHAR0) for i in prompt_ids if CHAR0 <= int(i) < 151643)
        r = int(_ROBOT_RE.search(text).group(1))
        ans = self.answers[r][self.count[r] % len(self.answers[r])]
        self.count[r] += 1
        return r, ans, 1000 * r + self.count[r]


class ScriptedReferenceModel:
    """The three model calls of the reference agent for one robot."""

    def __init__(self, answers, log):
        self.script, self.log, self.tag = _Answers(answers), log, None

    def eval(self):
        return self

    def to(self, device):
        return self

    def generate(self, input_ids=None, max_new_tokens=128, do_sample=False, return_dict_in_generate=True, **inputs):
        _, ans, self.tag = self.script.next(input_ids[0].tolist())
        seq = torch.cat([input_ids, torch.tensor([[CHAR0 + ord(c) for c in ans] + [EOS]])], dim=1)
        return SimpleNamespace(sequences=seq, past_key_values=None)

    def generate_latents(self, output_ids, pixel_values, image_grid_thw):
        return torch.tensor([[[float(self.tag)]]])

    def generate_traj(self, traj_latents, images_dp, depths_dp=None):
        tag = int(traj_latents.reshape(-1)[0])
        d = s1_digest(images_dp)
        self.log.append({"s1": tag, "frames": d})
        return trajectory(tag, d)


class ScriptedBatchedModel:
    """`generate_with_latents` / `generate_traj` of internnav_b200.internvla_n1.InternVLAN1ForCausalLM for B robots."""

    has_system1 = True
    config = SimpleNamespace(system1="nextdit_async", n_query=1)

    def __init__(self, answers, log):
        self.script, self.log = _Answers(answers), log
        self.device = torch.device("cpu")

    def generate_with_latents(self, prompts, pixel_values, image_grid_thw, max_new_tokens=128, **kw):
        gen, tags = [], []
        for p in prompts:
            _, ans, tag = self.script.next(p)
            gen.append([CHAR0 + ord(c) for c in ans] + [EOS])
            tags.append(float(tag))
        return SimpleNamespace(generated=gen, latents=torch.tensor(tags).reshape(-1, 1, 1), sequences=None)

    def generate_traj(self, traj_latents, images_dp, depths_dp=None, x_init=None):
        out = []
        for b in range(traj_latents.shape[0]):
            tag, d = int(traj_latents[b].reshape(-1)[0]), s1_digest(images_dp[b:b + 1])
            self.log.append({"s1": tag, "frames": d})
            out.append(trajectory(tag, d))
        return torch.cat(out).to(images_dp.device)


# ------------------------------------------------------------------------------------------------ replay of the traces
def make_agent(traces, device="cpu", x_init=None):
    """A batched agent serving one robot per trace (env j = traces[j]) on the scripted batched model -> (agent, log)."""
    from internnav_b200.agent_realworld import InternVLAN1AsyncAgent
    log = []
    model = ScriptedBatchedModel({t["case"]["robot"]: t["answers"] for t in traces}, log)
    c = traces[0]["case"]
    assert all((t["case"]["num_history"], t["case"]["resize"]) == (c["num_history"], c["resize"]) for t in traces)
    args = SimpleNamespace(device=device, model_path=None, resize_w=c["resize"], resize_h=c["resize"],
                           num_history=c["num_history"], plan_step_gap=[t["case"]["plan_step_gap"] for t in traces])
    return InternVLAN1AsyncAgent(args, model=model, processor=ScriptedProcessor(log), num_envs=len(traces),
                                 x_init=x_init), log


def _recorded(out):
    if isinstance(out, Exception):
        return {"error": type(out).__name__}
    return {"output": {"action": out.output_action, "pixel": out.output_pixel,
                       "trajectory": None if out.output_trajectory is None else np.asarray(out.output_trajectory).tolist()}}


def replay_steps(trace, device="cpu"):
    """Drive one robot through `step` exactly as the trace's server loop drove the reference; assert every output and
    model call.  -> the agent."""
    agent, log = make_agent([trace], device)
    case, ins = trace["case"], instruction(trace["case"]["robot"])
    for f in trace["frames"]:
        rgb, depth = frame(case["seed"], f["k"])
        if f["reset"]:
            agent.reset([0])
        for st in f["steps"]:
            del log[:]
            out = agent.step([0], [rgb], [depth], [np.eye(4)], [ins], None, [st["look_down"]])[0]
            want = {k: v for k, v in st.items() if k in ("output", "error")}
            assert _recorded(out) == want, (case, f["k"], st["look_down"])
            got = [dict(c, look_down=st["look_down"]) if "s2" in c else c for c in log]
            assert got == st["calls"], (case, f["k"], st["look_down"])
    return agent


def _robot_of(call):
    return int(_ROBOT_RE.search(call["s2"]).group(1)) if "s2" in call else call["s1"] // 1000


def replay_serve(traces, device="cpu", check_calls=None):
    """All traces side by side through `serve` (robot j = traces[j], resets where the traces have them; a robot whose
    trace has ended drops out); assert each robot's results and model calls.  check_calls(agent, calls_before) runs
    after every served frame.  -> the agent."""
    agent, log = make_agent(traces, device)
    for k in range(max(len(t["frames"]) for t in traces)):
        live = [j for j, t in enumerate(traces) if k < len(t["frames"])]
        fr = [traces[j]["frames"][k] for j in live]
        obs = [frame(traces[j]["case"]["seed"], k) for j in live]
        del log[:]
        before = dict(agent.calls)
        res = agent.serve(live, [o[0] for o in obs], [o[1] for o in obs],
                          [instruction(traces[j]["case"]["robot"]) for j in live], resets=[f["reset"] for f in fr])
        if check_calls is not None:
            check_calls(agent, before)
        for j, f, r in zip(live, fr, res):
            robot = traces[j]["case"]["robot"]
            got = {"error": type(r).__name__} if isinstance(r, Exception) else r
            assert got == f["result"], (traces[j]["case"], k)
            want = [{a: b for a, b in c.items() if a != "look_down"} for st in f["steps"] for c in st["calls"]]
            assert [c for c in log if _robot_of(c) == robot] == want, (traces[j]["case"], k)
    return agent
