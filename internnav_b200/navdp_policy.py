"""Mirror of the stand-alone NavDP policy (SURVEY.md §8f-3): `NavDPNet`,
internnav/model/basemodel/navdp/navdp_policy.py L40-339, on the same kernels as the InternVLA-N1 System-1 head.

What differs from the N1 head (all handled inside libn1b200.so, `n1_navdp_policy_load`): `RGBDBackbone` looks at
`memory_size` (8) RGB frames and ONE depth frame (navdp_backbone.py L205-283), the condition row is
[time, goal, goal, goal, 128 memory tokens] with LearnablePositionalEncoding tables, the sampler runs 10 DDPM steps over a
horizon of 24, and a critic head ranks the sampled trajectories (`predict_critic`, cross-attention restricted to the memory
tokens).  The reference runs this model in fp32; the kernels are bf16 with fp32 accumulation (parity is stated against the
fp32 oracle with the bf16-eager bound, like every other stage).  Inference entry points only: `forward` (the training loss
with image / pixel goals) is not built.
"""
import ctypes

import torch

from . import _bwd, _lib
from ._lib import OP_DENOISE, OP_RGBD, NavdpPolicyDims, TensorDesc, c_void_p, check
from .navdp import NavDP_Policy_DPT_CriticSum_DAT


_RENAME = {
    "rgbd_encoder.former_query.position_embedding.weight": "rgbd_encoder.former_query.weight",
    "rgbd_encoder.former_pe.position_embedding.weight": "rgbd_encoder.former_pe.weight",
}


class NavDPNet(NavDP_Policy_DPT_CriticSum_DAT):
    def __init__(self, image_size=224, memory_size=8, predict_size=24, temporal_depth=16, heads=8, token_dim=384,
                 device="cuda:0"):
        super().__init__(image_size=image_size, memory_size=memory_size, predict_size=predict_size,
                         temporal_depth=temporal_depth, heads=heads, token_dim=token_dim, device=device)
        self.num_train_timesteps = 10   # DDPMScheduler(num_train_timesteps=10, ...) navdp_policy.py L119-121
        self.model_name = "NavDPNet"
        self._point = None

    # ------------------------------------------------------------------ weights
    def _load(self, sd):
        L = _lib.lib()
        dev = self._device
        if dev.type != "cuda":
            raise RuntimeError("n1b200 has no CPU path: construct NavDPNet with device='cuda:N'")
        flat = {}
        for k, v in sd.items():
            if not torch.is_tensor(v) or not v.is_floating_point():
                continue
            k = _RENAME.get(k, k)
            if k == "cond_pos_embed.position_embedding.weight":
                k, v = "cond_pos_embed", v.unsqueeze(0)
            elif k == "out_pos_embed.position_embedding.weight":
                k, v = "out_pos_embed", v.unsqueeze(0)
            # the image / pixel goal encoders and the auxiliary heads serve `forward` (training) only
            if k.startswith(("image_encoder.", "pixel_encoder.", "pixel_aux_head.", "image_aux_head.")):
                continue
            flat[k] = v
        self._point = (flat["point_encoder.weight"].detach().to(dev, torch.float32).contiguous(),
                       flat["point_encoder.bias"].detach().to(dev, torch.float32).contiguous())
        h = c_void_p()
        check(L.n1_create(ctypes.byref(h), dev.index or 0))
        keep, descs = [], []
        for name, t in flat.items():
            t = t.detach().to(dev, torch.float32 if t.dtype not in (torch.float32, torch.bfloat16) else t.dtype).contiguous()
            keep.append(t)
            d = TensorDesc()
            d.name, d.data, d.dtype = name.encode(), t.data_ptr(), _lib.dtype_code(t)
            d.ndim = min(t.dim(), 4)
            for i, s in enumerate(list(t.shape)[:4]):
                d.shape[i] = s
            descs.append(d)
        arr = (TensorDesc * len(descs))(*descs)
        dims = NavdpPolicyDims(self.token_dim, self.attention_heads, self.temporal_depth, self.predict_size,
                               self.memory_size, 1, 3, self.num_train_timesteps)
        with torch.cuda.device(dev):
            check(L.n1_navdp_policy_load(h, ctypes.byref(dims), arr, len(descs), _lib.stream_ptr()))
            torch.cuda.synchronize()
        if self._handle is not None:
            L.n1_destroy(self._handle)
        self._handle = h
        del keep

    # ------------------------------------------------------------------ reference API
    def rgbd_encoder(self, images, depths):
        """RGBDBackbone.forward (navdp_backbone.py L246-283): images [B, memory_size, 224, 224, 3] in [0, 1], depths
        [B, 1, 224, 224(, 1)] metres -> memory tokens [B, 16 * memory_size, 384]."""
        B = images.shape[0]
        if tuple(images.shape[1:]) != (self.memory_size, 224, 224, 3) or depths.shape[0] != B or depths.shape[1] != 1:
            raise ValueError("NavDPNet.rgbd_encoder takes images [B, %d, 224, 224, 3] and depths [B, 1, 224, 224(, 1)]; got "
                             "%s and %s" % (self.memory_size, tuple(images.shape), tuple(depths.shape)))
        rgb = images.to(self._device, torch.float32).contiguous()
        dep = depths.to(self._device, torch.float32).reshape(B, 1, 224, 224).contiguous()
        out = torch.empty(B, 16 * self.memory_size, self.token_dim, device=self._device, dtype=torch.bfloat16)
        ws, n = self._scratch(OP_RGBD, B)
        check(_lib.lib().n1_rgbd_encode(self._h(), _lib.ptr(ws), n, _lib.ptr(rgb), _lib.ptr(dep), _lib.ptr(out), B,
                                       _lib.stream_ptr()))
        return out

    def point_encoder(self, goal_point):
        """nn.Linear(3, 384) on the goal point (navdp_policy.py L87): [B, 3] -> [B, 384] (small fp32 product kernel)."""
        g = torch.as_tensor(goal_point, dtype=torch.float32).to(self._device).reshape(-1, 3).contiguous()
        return _bwd.sgemm(g, self._point[0], trans_b=True) + self._point[1]

    def predict_critic(self, predict_trajectory, rgbd_embed):
        """navdp_policy.py L172-187: trajectories [B * Ns, T, 3] -> critic values [B * Ns] (fp32)."""
        B = rgbd_embed.shape[0]
        R, T, _ = predict_trajectory.shape
        x = predict_trajectory.to(self._device, torch.float32).contiguous()
        rgbd = rgbd_embed.to(self._device, torch.bfloat16).contiguous()
        out = torch.empty(R, device=self._device, dtype=torch.float32)
        ws, n = self._scratch(OP_DENOISE, B, R // B, T)
        check(_lib.lib().n1_navdp_critic(self._h(), _lib.ptr(ws), n, _lib.ptr(x), _lib.ptr(rgbd), _lib.ptr(out), B, R // B, T,
                                        _lib.stream_ptr()))
        return out

    def _sample_and_rank(self, goal_embed, rgbd_embed, sample_num, x_init, step_noise):
        B = rgbd_embed.shape[0]
        if x_init is None:
            x_init = torch.randn((sample_num * B, self.predict_size, 3), device=self._device)
            step_noise = torch.randn((self.num_train_timesteps - 1, sample_num * B, self.predict_size, 3), device=self._device)
        naction = self.sample(goal_embed, rgbd_embed, x_init, step_noise, num_steps=self.num_train_timesteps)
        critic_values = self.predict_critic(naction, rgbd_embed)
        traj = torch.cumsum(naction / 4.0, dim=1)
        # the reference ranks over ALL samples of the call (navdp_policy.py L320-321, L337-338)
        negative_trajectory = traj[critic_values.argsort()[0:8]]
        positive_trajectory = traj[(-critic_values).argsort()[0:8]]
        return negative_trajectory, positive_trajectory

    def predict_pointgoal_batch_action_vel(self, goal_point, input_images, input_depths, sample_num=32, x_init=None,
                                           step_noise=None):
        """navdp_policy.py L302-322.  `x_init` [Ns*B, T, 3] / `step_noise` [K-1, Ns*B, T, 3] inject the sampler's draws."""
        with torch.no_grad():
            rgbd_embed = self.rgbd_encoder(input_images, input_depths)
            goal = self.point_encoder(goal_point).unsqueeze(1).to(torch.bfloat16)
            return self._sample_and_rank(goal, rgbd_embed, sample_num, x_init, step_noise)

    def predict_nogoal_batch_action_vel(self, input_images, input_depths, sample_num=32, x_init=None, step_noise=None):
        """navdp_policy.py L324-339: zero goal embedding."""
        with torch.no_grad():
            rgbd_embed = self.rgbd_encoder(input_images, input_depths)
            goal = torch.zeros(rgbd_embed.shape[0], 1, self.token_dim, device=self._device, dtype=torch.bfloat16)
            return self._sample_and_rank(goal, rgbd_embed, sample_num, x_init, step_noise)

    # the N1-only pieces of the parent class do not exist on this model
    def goal_embed(self, vlm_tokens):
        raise NotImplementedError("NavDPNet has no VLM goal path (that is the InternVLA-N1 head)")

    predict_pointgoal_action_async = goal_embed
    forward_vlm_traj = goal_embed
    rgb_memory_tokens = goal_embed
