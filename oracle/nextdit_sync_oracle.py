"""CPU restatement of the reference's synchronous NextDiT System 1 (`system1 = "nextdit"`) -- TEST INFRASTRUCTURE, not
product code.

internvla_n1.py L359-432 with `'async' not in system1`: the condition tokens are `cond_projector(traj_latents)` alone
(L361, L380-381: no DINOv2 / MemoryEncoder / QFormer, `images_dp` unused), then the same CFG batch and flow-matching
Euler loop over the same trajectory DiT as the asynchronous head.  The DiT, the action encoder / decoder and the
scheduler are oracle/nextdit_oracle.py's; this file adds only the synchronous conditioning and the loop around it.
State-dict keys: internnav_b200.manifest.nextdit_shapes(asynchronous=False)."""
import torch
import torch.nn.functional as F

from . import nextdit_oracle as O


def condition_tokens(sd, traj_latents):
    """internvla_n1.py L361, L380-381: [B, n_query, 3584] -> [B, n_query, 768]."""
    return O._lin(sd, "cond_projector.2", F.gelu(O._lin(sd, "cond_projector.0", traj_latents), approximate="tanh"))


def generate_traj(sd, traj_latents, x_init, guidance_scale=1.0, num_inference_steps=10, num_sample_trajs=32):
    """internvla_n1.py L359-432 for system1 = "nextdit".  x_init replaces `randn_tensor` (L389-394): [B * Ns, 32, 3]."""
    dtype = traj_latents.dtype
    hidden = condition_tokens(sd, traj_latents)
    hidden_in = torch.cat((torch.zeros_like(hidden), hidden), 0).repeat_interleave(num_sample_trajs, dim=0)
    timesteps, sigmas = O.flow_match_schedule(num_inference_steps)
    latents = x_init.to(dtype)
    for i, t in enumerate(timesteps):
        inp = O.action_features(sd, latents).repeat(2, 1, 1)
        tt = t.unsqueeze(0).expand(inp.shape[0]).to(inp.device, torch.long)
        pred = O._lin(sd, "action_decoder", O.traj_dit(sd, inp, tt, hidden_in))
        uncond, cond = pred.chunk(2)
        pred = uncond + guidance_scale * (cond - uncond)
        latents = (latents.to(torch.float32) + (sigmas[i + 1] - sigmas[i]).to(pred.device) * pred).to(pred.dtype)
    return latents
