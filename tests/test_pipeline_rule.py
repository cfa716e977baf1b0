"""The parity-wait rule of the plane-gather kernels (DESIGN.md §3.5) replayed under random schedules on the host
(tools/pipeline_sim.py): the producer counts the host code chooses, with the two consumer warpgroups that each consume
every slot, never deadlock or consume a stale stage; the two earlier multi-issuer configurations that hung / corrupted
tiles on the GPU fail here too."""
import os
import sys

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import pipeline_sim as ps  # noqa: E402


@pytest.mark.parametrize("stages", [2, 3, 4, 5, 6, 7, 8])
def test_host_chosen_role_counts_are_sound(stages):
    for nunits in (1, 2, 3, 4, 6, 8):
        Wu = ps.producer_choice(stages)
        assert stages % Wu == 0
        res = {ps.sim(Wu, nunits, stages, 2, 6, seed, every=True) for seed in range(6)}
        assert res == {"ok"}, (Wu, nunits, stages, res)


def test_rule_violations_fail_in_the_replay():
    assert "DEADLOCK" in {ps.sim(7, 8, 8, 2, 14, s) for s in range(8)}       # 7 producers on 8 stages, 2 issuers (bf16 wgrad hang)
    assert {ps.sim(6, 8, 6, 4, 14, s) for s in range(12)} != {"ok"}           # 4 issuers on a 6-stage ring (wrong tiles)
