"""Differential tests against the reference's OWN classes on seeded random scenarios (oracle/live_traces.py), beyond the
committed step-by-step goldens:

  * InternVLAN1Net host logic (s2_step / step_no_infer / s1_step_latent / reset) vs internnav_b200.policy.InternVLAN1Policy
  * InternVLAN1Agent (real S2 worker thread, polling sleeps shortened) vs internnav_b200.agent.InternVLAN1Agent

The reference's traces were recorded by oracle/gen_golden_live.py into tests/golden/live_reference_traces.json, so the
comparison runs everywhere, entry by entry.  Where the reference tree is installed it is also run live.
"""
import json
import os

import pytest

from oracle import live_traces as T, ref_loader

with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "live_reference_traces.json")) as fh:
    GOLD = json.load(fh)


def _same(ref, mine):
    mine = json.loads(json.dumps(mine))  # tuples -> lists, as the stored traces have them
    for k, (a, b) in enumerate(zip(ref, mine)):
        assert a == b, "trace entry %d" % k
    assert len(ref) == len(mine)


@pytest.mark.parametrize("seed", T.POLICY_SEEDS)
def test_policy_host_logic_vs_live_reference(seed):
    mine = T.policy_trace(seed)
    _same(GOLD["policy:%d" % seed], mine)
    if ref_loader.available():
        _, Net = ref_loader.load_reference_policy()
        _same(json.loads(json.dumps(T.policy_trace(seed, Net))), mine)


@pytest.mark.parametrize("seed,mode", T.AGENT_CASES)
def test_agent_vs_live_reference(seed, mode):
    mine = T.agent_trace(seed, mode)
    _same(GOLD["agent:%d:%s" % (seed, mode)], mine)
    if ref_loader.available():
        _same(json.loads(json.dumps(T.agent_trace(seed, mode, ref_loader.load_reference_agent))), mine)
