"""CPU checks of the fused NavDP decoder attention blocks (dec_attn_block.cu); tests/test_no_spills_host.py holds both
kernels to zero spill.

The float64 reference and bound of tests/test_dec_blocks_gpu.py must accept the correct result and reject what a kernel
with a causal mask shifted by one key, a trajectory boundary off by one row, or a tile reading the neighbouring
environment's K / V would compute."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_dec_blocks_gpu as G  # noqa: E402
from test_hopper_kernels_gpu import bound_violations  # noqa: E402


def _rejects(ref, bound, wrong):
    """The correct result rounded to bf16 passes; the wrong one fails somewhere."""
    bad, _ = bound_violations(ref.to(torch.bfloat16), ref, bound)
    assert not bool(bad.any())
    bad, _ = bound_violations(wrong.to(torch.bfloat16), ref, bound)
    return int(bad.sum())


@pytest.mark.parametrize("T", [8, 17])
def test_bound_rejects_a_causal_mask_shifted_by_one_key(T):
    B, Ns = 1, 3
    p, x = G.make_params(True, 1), G.make_x(B * Ns * T, 2)
    ref, bound = G.sa_ref(x, p, B, Ns, T, True)
    wrong, _ = G.sa_ref(x, p, B, Ns, T, True, key_shift=1)
    assert _rejects(ref, bound, wrong) > 0


@pytest.mark.parametrize("shift", [1, -1])
def test_bound_rejects_a_trajectory_boundary_off_by_one_row(shift):
    B, Ns, T = 1, 3, 8
    p, x = G.make_params(True, 3), G.make_x(B * Ns * T, 4)
    ref, bound = G.sa_ref(x, p, B, Ns, T, True)
    wrong, _ = G.sa_ref(x, p, B, Ns, T, True, row_shift=shift)
    assert _rejects(ref, bound, wrong) > 0


def test_bound_rejects_a_tile_reading_the_neighbouring_environments_kv():
    B, Ns, T, mtok = 2, 2, 8, 34
    p, x, kv = G.make_params(False, 5), G.make_x(B * Ns * T, 6), G.make_kv(B, mtok, 7)
    ref, bound = G.ca_ref(x, p, kv, mtok, B, Ns, T)
    wrong, _ = G.ca_ref(x, p, kv, mtok, B, Ns, T, env_shift=1)
    n = _rejects(ref, bound, wrong)
    assert n > 0
    # only environment 0's rows are wrong
    bad, _ = bound_violations(wrong.to(torch.bfloat16), ref, bound)
    assert not bool(bad[Ns * T:].any())
