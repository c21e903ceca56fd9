"""Tail of a System-1 step: trajectories -> discrete action ids.

Mirrors internnav/model/utils/vln_utils.py (`traj_to_actions` L63-136, `chunk_token` L36-60) and the list clean-up in
InternVLAN1Net.s1_step_latent (internvla_n1_policy.py L207-214).  Integer results: bit-exact for identical inputs.

Product path: `batched_traj_to_actions` on CUDA tensors runs the library kernel (n1_traj_to_actions, csrc/postprocess.cu:
float32 cumsum, float64 mean, pure pursuit -- one block per environment) and copies back only the ids.  The numpy
functions below keep the reference function's contract for host tensors (`traj_to_actions` is what the reference's
callers import) and are the checker of the kernel in tests/test_postprocess_gpu.py.
"""
import ctypes

import numpy as np
import torch


def _discretise(trajectory, step_size=0.25, turn_angle_deg=15, lookahead=4, max_actions=None):
    """`max_actions`: stop once that many ids exist.  The loop only ever appends, so the first `max_actions` entries are
    identical to those of the full run -- which is all `s1_step_latent` keeps (internvla_n1_policy.py L212-214)."""
    actions = []
    yaw = 0.0
    pos = trajectory[0]
    turn_angle_rad = np.deg2rad(turn_angle_deg)
    goal = trajectory[-1]

    def normalize_angle(angle):
        return (angle + np.pi) % (2 * np.pi) - np.pi

    while np.linalg.norm(pos - goal) > 0.2:
        if max_actions is not None and len(actions) >= max_actions:
            break
        dists = np.linalg.norm(trajectory - pos, axis=1)
        nearest_idx = np.argmin(dists)
        target = trajectory[min(nearest_idx + lookahead, len(trajectory) - 1)]
        target_dir = target - pos
        if np.linalg.norm(target_dir) < 1e-6:
            break
        delta_yaw = normalize_angle(np.arctan2(target_dir[1], target_dir[0]) - yaw)
        n_turns = int(round(delta_yaw / turn_angle_rad))
        if n_turns > 0:
            actions += [2] * n_turns
        elif n_turns < 0:
            actions += [3] * (-n_turns)
        yaw = normalize_angle(yaw + n_turns * turn_angle_rad)
        next_pos = pos + step_size * np.array([np.cos(yaw), np.sin(yaw)])
        if np.linalg.norm(next_pos - goal) > np.linalg.norm(pos - goal):
            break
        actions.append(1)
        pos = next_pos
    return actions


def _mean_trajectory(a):
    """a: float32 numpy [Ns, T, 3] already divided by 4 in the first two channels."""
    n, t = a.shape[0], a.shape[1]
    xy = np.zeros((n, t + 1, 2))
    xy[:, 1:] = np.cumsum(a[:, :, :2], axis=1)
    return np.mean(xy, axis=0)


def traj_to_actions(dp_actions, use_discrate_action=True):
    """Same contract as the reference function, including the in-place `/= 4` on the caller's tensor."""
    dp_actions[:, :, :2] /= 4.0
    traj = _mean_trajectory(dp_actions.float().cpu().numpy())
    return _discretise(traj) if use_discrate_action else traj


def batched_traj_to_actions_gpu(dp_actions, num_envs, max_actions=None, cap=64, return_mean=False):
    """dp_actions CUDA [num_envs * Ns, T, 3] (not modified) -> list of per-environment action lists through the library
    kernel; D2H = num_envs * (cap + 1) int32.  Lists longer than `cap` are refused (cannot happen with max_actions <= 4:
    one walk iteration appends at most 12 turns + 1 forward)."""
    from . import _lib
    assert dp_actions.is_cuda and dp_actions.dim() == 3 and dp_actions.shape[2] == 3 and dp_actions.shape[0] % num_envs == 0
    t = dp_actions.detach().float().contiguous()
    ns, T = t.shape[0] // num_envs, t.shape[1]
    ids = torch.empty(num_envs, cap, dtype=torch.int32, device=t.device)
    cnt = torch.empty(num_envs, dtype=torch.int32, device=t.device)
    mean = torch.empty(num_envs, T + 1, 2, dtype=torch.float64, device=t.device) if return_mean else None
    _lib.check(_lib.lib().n1_traj_to_actions(_lib.ptr(t), num_envs, ns, T, ctypes.c_double(float(np.deg2rad(15))),
                                             ctypes.c_double(0.25), 4, int(max_actions or 0), cap, _lib.ptr(ids),
                                             _lib.ptr(cnt), _lib.ptr(mean), _lib.stream_ptr()))
    host = torch.cat((ids, cnt[:, None]), dim=1).cpu().numpy()       # the one D2H of the tail
    out = []
    for e in range(num_envs):
        n = int(host[e, cap])
        if n > cap:
            raise RuntimeError("action list of environment %d has %d ids (> cap %d)" % (e, n, cap))
        out.append(host[e, :n].tolist())
    return (out, mean) if return_mean else out


def batched_traj_to_actions(dp_actions, num_envs, use_discrate_action=True, max_actions=None):
    """dp_actions [num_envs * Ns, T, 3] (not modified) -> list of per-environment action lists (optionally only their
    first `max_actions` entries, see _discretise).  CUDA tensors take the kernel path; host tensors the numpy one."""
    if torch.is_tensor(dp_actions) and dp_actions.is_cuda and use_discrate_action:
        return batched_traj_to_actions_gpu(dp_actions, num_envs, max_actions=max_actions)
    a = dp_actions.detach().float().cpu().numpy().copy()
    a[:, :, :2] /= 4.0
    ns = a.shape[0] // num_envs
    out = []
    for e in range(num_envs):
        traj = _mean_trajectory(a[e * ns:(e + 1) * ns])
        out.append(_discretise(traj, max_actions=max_actions) if use_discrate_action else traj)
    return out


def batched_traj_to_waypoints(dp_actions, num_envs):
    """dp_actions [num_envs * Ns, T, 3] (not modified) -> float64 numpy [num_envs, T + 1, 2]: per environment the mean path
    that `traj_to_actions(..., use_discrate_action=False)` returns (the real-world agent's System-1 output, vln_utils.py
    L127-133), bit-equal to it.  CUDA tensors take the kernel (n1_traj_mean_path; D2H = the paths); host tensors numpy."""
    assert dp_actions.dim() == 3 and dp_actions.shape[2] == 3 and dp_actions.shape[0] % num_envs == 0
    if not dp_actions.is_cuda:
        return np.stack(batched_traj_to_actions(dp_actions, num_envs, use_discrate_action=False))
    from . import _lib
    t = dp_actions.detach().float().contiguous()
    ns, T = t.shape[0] // num_envs, t.shape[1]
    mean = torch.empty(num_envs, T + 1, 2, dtype=torch.float64, device=t.device)
    _lib.check(_lib.lib().n1_traj_mean_path(_lib.ptr(t), num_envs, ns, T, _lib.ptr(mean), _lib.stream_ptr()))
    return mean.cpu().numpy()


def chunk_token(dp_actions):
    out_list = []
    for i in range(len(dp_actions)):
        xyyaw = dp_actions[i]
        x, yaw = xyyaw[0], xyyaw[-1]
        x_prop = torch.abs(x / 0.25)
        yaw_prop = torch.abs(yaw * 12 / torch.pi)
        if x < 0.05 and torch.abs(yaw) < 0.05:
            out_list.append(0)
        elif x_prop >= yaw_prop:
            out_list.append(1)
        elif yaw < 0:
            out_list.append(3)
        else:
            out_list.append(2)
    return out_list


def s1_action_list(action_list):
    """internvla_n1_policy.py L212-214: drop zeros, keep the first 4."""
    return [x for x in action_list if x != 0][:4]
