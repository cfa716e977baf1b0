"""The parity-wait rule (DESIGN.md §3.5) with convolution consumers that keep one wgmma group in flight: each consumer
warpgroup releases slot n - 1 (and the weight stage, after its last tile) only once it has taken slot n.  Replayed
under random schedules (tools/pipeline_sim.py, lag=True) for every A-ring depth (sa) and weight-ring depth (sb) the host
code can pick, with the producer assignments of both convolution kernels.  The kernels' own bookkeeping is exercised by
the GPU tests."""
import os
import sys

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import pipeline_sim as ps  # noqa: E402


@pytest.mark.parametrize("sa", [3, 4, 5, 6, 7, 8])
@pytest.mark.parametrize("sb", [2, 3])
@pytest.mark.parametrize("kernel", ["k_conv_pl", "k_conv_tc"])
def test_conv_roles_with_lagged_release_are_sound(kernel, sb, sa):
    # k_conv_pl: W = min(8, sa) = sa producer warps, each owning one stage; k_conv_tc: every gather warp fills every
    # slot (one producer that walks every stage).  T = 1, 2 or 4 tiles share a weight stage.
    W = sa if kernel == "k_conv_pl" else 1
    for T in (1, 2, 4):
        res = {ps.sim(W, T, sa, 2, 6, seed, every=True, lag=True, gbufs=sb) for seed in range(6)}
        assert res == {"ok"}, (kernel, sa, sb, T, res)
