"""Generate tests/golden/nextdit_sync_reference.npz by running the REFERENCE's own `generate_traj` for the synchronous
head (`system1 = "nextdit"`, internvla_n1.py L359-432) -- TEST INFRASTRUCTURE, runs only where /root/reference exists.

Recorded the way oracle/gen_golden_nextdit.py records nextdit_reference.npz: the reference method is called unbound on a
stand-in `self`, which here carries the modules the reference's own InternVLAN1MetaModel.__init__ builds for
system1 = "nextdit" (internvla_n1_arch.py L121-140: traj_dit, action_encoder / decoder, pos_encoding, cond_projector; no
RGB branch), with the `diffusers` leaf modules of oracle/diffusers_standin.py and the seeded x_init injected for
`randn_tensor`.  Weights: internnav_b200.manifest.random_nextdit_state_dict(5, asynchronous=False), loaded with every key
used (the reference's `latent_queries` and `freqs_cis` buffers are the only tensors it does not receive).  One environment,
3 trajectories, guidance 1.0 and 2.5; also the condition tokens.

Usage:  python -m oracle.gen_golden_nextdit_sync"""
import importlib
import os
import sys
import types

import numpy as np
import torch
import torch.nn as nn

from .gen_golden_nextdit import B, NS, SEED, make_inputs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def reference_meta_model(system1):
    """The modules the reference's InternVLAN1MetaModel.__init__ builds for `system1` (internvla_n1_arch.py L121-145; None:
    no system1 in the config), on a bare nn.Module base instead of the 7B Qwen2_5_VLModel."""
    from . import ref_loader
    ref_loader.load_reference_nextdit()
    arch = importlib.import_module("internnav.model.basemodel.internvla_n1.internvla_n1_arch")

    class Base(nn.Module):
        def __init__(self, config):
            super().__init__()

    class Model(arch.InternVLAN1MetaModel, Base):
        pass

    cfg = types.SimpleNamespace(n_query=4, hidden_size=3584)
    if system1 is not None:
        cfg.system1 = system1
    return Model(cfg)


def build_reference_sync_model(sd):
    """-> (reference module, generate_traj, stand-in self, model) for system1 = "nextdit" with the weights of `sd`."""
    from . import ref_loader
    ref_loader.load_reference_nextdit()
    tu = types.ModuleType("diffusers.utils.torch_utils")
    tu.randn_tensor = lambda *a, **k: None      # replaced per call
    sys.modules["diffusers.utils.torch_utils"] = tu
    sys.modules["diffusers.utils"].torch_utils = tu
    main = importlib.import_module("internnav.model.basemodel.internvla_n1.internvla_n1")
    model = reference_meta_model("nextdit").eval()
    missing, unexpected = model.load_state_dict(sd, strict=False)
    assert not unexpected and all("freqs_cis" in k or k == "latent_queries" for k in missing), (missing, unexpected)

    class Self:
        def get_system1_type(self):
            return "nextdit"

        def get_model(self):
            return model

    return main, main.InternVLAN1ForCausalLM.generate_traj, Self(), model


def main():
    sys.path.insert(0, ROOT)
    from internnav_b200.manifest import random_nextdit_state_dict
    sd = random_nextdit_state_dict(SEED, asynchronous=False)
    mod, generate_traj, self_, model = build_reference_sync_model(sd)
    inp = make_inputs()
    out = {}
    for scale in (1.0, 2.5):
        mod.randn_tensor = lambda shape, generator=None, device=None, dtype=None: inp["x_init"].to(dtype).clone()
        with torch.no_grad():
            out[scale] = generate_traj(self_, inp["traj_latents"], inp["images_dp"], guidance_scale=scale,
                                       num_sample_trajs=NS)
    with torch.no_grad():
        cond = model.cond_projector(inp["traj_latents"])
    path = os.path.join(ROOT, "tests", "golden", "nextdit_sync_reference.npz")
    np.savez_compressed(path, seed=SEED, batch=B, ns=NS, traj_scale_1=out[1.0].numpy(), traj_scale_2p5=out[2.5].numpy(),
                        condition_tokens=cond.numpy())
    print("wrote", path, {k: tuple(v.shape) for k, v in out.items()}, cond.shape)


if __name__ == "__main__":
    main()
