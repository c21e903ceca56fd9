"""The reference's two registries, for code that builds the policy and the agent from configuration
(SURVEY.md §8b): `Agent.register('internvla_n1')` / `Agent.init(AgentCfg)` (internnav/agent/base.py L18-37,
internvla_n1_agent.py L21-43) and `get_policy('InternVLAN1_Policy')` / `get_config(...)`
(internnav/model/__init__.py L18-24, L50-56).

`model_settings` keys follow scripts/eval/configs/h1_internvla_n1_async_cfg.py: model_path, device, width / height /
hfov, resize_w / resize_h, num_history, continuous_traj, infer_mode, sys2_max_forward_step, env_num (number of
environments this agent serves; the reference supports 1), max_new_tokens is fixed at 128 by the policy (L171).
"""
from types import SimpleNamespace

from .agent import InternVLAN1Agent
from .internvla_n1 import InternVLAN1ForCausalLM
from .policy import InternVLAN1Policy


class InternVLAN1ModelConfig(SimpleNamespace):
    """`InternVLAN1ModelConfig(model_cfg={'model': {...}})` (internvla_n1.py L24-29), reduced to what the policy reads."""

    def __init__(self, model_cfg=None, **kw):
        super().__init__(model_cfg=model_cfg, **kw)


class InternVLAN1Net(InternVLAN1Policy):
    """Config-driven construction of the batched policy, as `get_policy(name)(config=get_config(name)(model_cfg=...))`
    does for the reference class (internvla_n1_agent.py L39-43, internvla_n1_policy.py L29-57)."""

    def __init__(self, config, model=None, processor=None):
        m = dict(config.model_cfg["model"])
        device = m.get("device", "cuda:0")
        if model is None:
            model = InternVLAN1ForCausalLM.from_pretrained(m["model_path"], device_map={"": device})
        if processor is None:  # the reference's own collaborators (policy L44-47)
            from transformers import AutoProcessor, AutoTokenizer
            processor = AutoProcessor.from_pretrained(m["model_path"])
            processor.tokenizer = AutoTokenizer.from_pretrained(m["model_path"], use_fast=True)
            processor.tokenizer.padding_side = "left"
        super().__init__(model, processor, num_envs=int(m.get("env_num", 1)), num_history=int(m.get("num_history", 8)),
                         resize_w=int(m.get("resize_w", 384)), resize_h=int(m.get("resize_h", 384)),
                         continuous_traj=bool(m.get("continuous_traj", True)), device=device)
        # the System 1 is the checkpoint's (config.json `system1`); a setting that names another one is an error
        system1 = getattr(getattr(model, "config", None), "system1", m.get("system1"))
        if m.get("system1", system1) != system1:
            raise ValueError("model_settings system1=%r, but the checkpoint at %s has system1=%r"
                             % (m["system1"], m["model_path"], system1))
        m["system1"] = system1
        self.model_config = SimpleNamespace(**m)


def get_policy(policy_name):
    if policy_name == "InternVLAN1_Policy":
        return InternVLAN1Net
    raise ValueError(f"Policy {policy_name} not found")  # the other policies of the reference are out of scope


def get_config(policy_name):
    if policy_name == "InternVLAN1_Policy":
        return InternVLAN1ModelConfig
    raise ValueError(f"Policy {policy_name} not found")


class Agent:
    """internnav/agent/base.py: a name -> class registry with `init(config)`."""
    agents = {}

    @classmethod
    def register(cls, agent_type):
        def decorator(agent_class):
            if agent_type in cls.agents:
                raise ValueError(f"Agent {agent_type} already registered.")
            cls.agents[agent_type] = agent_class
            return agent_class
        return decorator

    @classmethod
    def init(cls, config, **kw):
        return cls.agents[config.model_name](config, **kw)


@Agent.register("internvla_n1")
class ConfiguredInternVLAN1Agent(InternVLAN1Agent):
    """`InternVLAN1Agent(config: AgentCfg)` (internvla_n1_agent.py L29-85): everything comes from
    `config.model_settings`.  `policy=` / `preprocessor=` may be injected (tests; sharing one model between agents)."""

    def __init__(self, config, policy=None, preprocessor=None):
        s = dict(config.model_settings)
        self.config = config
        if policy is None:
            name = s.get("policy_name", "InternVLAN1_Policy")
            policy = get_policy(name)(config=get_config(name)(model_cfg={"model": s}))
        if hasattr(policy, "eval"):
            policy.eval()
        super().__init__(policy, num_envs=int(s.get("env_num", 1)), infer_mode=s.get("infer_mode", "sync"),
                         sys2_max_forward_step=int(s.get("sys2_max_forward_step", 8)), width=s.get("width", 640),
                         height=s.get("height", 480), hfov=s.get("hfov", 79), preprocessor=preprocessor)
