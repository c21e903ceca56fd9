"""The System-2 training calls refuse a continuation plan (a generation plan created over a K/V pool).  Such a plan's
rows live in the pool (slot * capacity + ...), while the training workspace's cache holds B * slot rows per layer: a
pool slot >= B would be written past that cache.  The refusal must come before any launch, whatever the workspace."""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
N1_ERR_ARG = -2  # include/n1b200.h


def test_train_refuses_continuation_plan():
    from internnav_b200 import _lib
    from internnav_b200.qwen import KVPool, System2
    from oracle import qwen_oracle as Q
    cfg = Q.tiny_cfg()
    s2 = System2(cfg, device="cuda:0")
    s2.load_state_dict(Q.make_s2_state_dict(cfg, seed=17))
    prompt = Q.make_prompt(np.random.Generator(np.random.PCG64(17)), 12, [], 5)
    L, h = _lib.lib(), s2._h()
    assert L.n1_s2_train_workspace_bytes(h, s2.llm_plan([prompt], [], 1)) > 0  # the same prompt without a pool trains

    pool = KVPool(s2, 3, 256)
    plan = s2.llm_plan([prompt], [], 1, pool=pool, reused=[0], slots=[2])  # B = 1, slot 2
    assert L.n1_s2_train_workspace_bytes(h, plan) == 0
    assert b"pool" in L.n1_last_error(), L.n1_last_error()
    ws = torch.zeros(256, dtype=torch.uint8, device="cuda")  # real, and too small for any training call
    nq, H = cfg["n_query"], cfg["hidden"]
    feats = torch.zeros(1, cfg["v_out"], dtype=torch.bfloat16, device="cuda")
    states = torch.zeros(1, nq, H, dtype=torch.bfloat16, device="cuda")
    rc = L.n1_s2_train_forward(h, plan, _lib.ptr(ws), ws.numel(), _lib.ptr(feats), _lib.ptr(states), _lib.stream_ptr())
    assert rc == N1_ERR_ARG and b"pool" in L.n1_last_error(), (rc, L.n1_last_error())
    grad_latent = torch.zeros(nq, H, dtype=torch.float32, device="cuda")
    rc = L.n1_s2_train_backward(h, plan, _lib.ptr(ws), ws.numel(), _lib.ptr(states), _lib.ptr(grad_latent),
                                _lib.stream_ptr())
    assert rc == N1_ERR_ARG and b"pool" in L.n1_last_error(), (rc, L.n1_last_error())
    torch.cuda.synchronize()
    assert not ws.any() and not states.any() and not grad_latent.any()
    assert pool.valid(2) == 0
