"""Record tests/golden/live_reference_traces.json: the traces that the REFERENCE's own InternVLAN1Net and
InternVLAN1Agent produce on the scenarios of oracle/live_traces.py.  Needs the reference tree (oracle/ref_loader.py).

    python -m oracle.gen_golden_live
"""
import json
import os

from oracle import live_traces as T, ref_loader


def main():
    _, Net = ref_loader.load_reference_policy()
    out = {"policy:%d" % s: T.policy_trace(s, Net) for s in T.POLICY_SEEDS}
    for s, mode in T.AGENT_CASES:
        out["agent:%d:%s" % (s, mode)] = T.agent_trace(s, mode, ref_loader.load_reference_agent)
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden",
                        "live_reference_traces.json")
    with open(path, "w") as fh:
        json.dump(out, fh, separators=(",", ":"), sort_keys=True)
        fh.write("\n")
    print(path)


if __name__ == "__main__":
    main()
