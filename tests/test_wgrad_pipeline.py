"""The weight-gradient kernels `k_wgrad_pl` and `k_wgrad_tc` keep one wgmma group in flight over a unit ring and a gout
ring (DESIGN.md §3.2), and a gout tile holds only the column blocks of the CTA's units.

* The built library's SASS must show a `wait_group 1` that follows a real MMA group (no GPU needed; see
  test_sass_retire.py for why an empty dummy group would drain every slot anyway).
* The lagged release order is replayed under random schedules (tools/pipeline_sim.py) for every unit-ring depth
  (3-8) and gout-ring depth (2-4) the host planner can pick, with 1 and 2 units per row tile, for both producer
  schemes: k_wgrad_pl's Wg gout warps plus Wu unit warps, and k_wgrad_tc's gather warps that walk one slot sequence.
* On the GPU, dW at Cout = 192 (two units of 64 columns per pass, whose column blocks are not adjacent) matches an
  fp64 reference for both kernels."""
import os
import re
import subprocess
import sys

import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import pipeline_sim as ps  # noqa: E402


@pytest.fixture(scope="module")
def sass():
    from pasco_b200 import build, _lib
    build.build()
    return subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout


@pytest.mark.parametrize("kernel", ["k_wgrad_pl", "k_wgrad_tc"])
def test_wgrad_consumers_wait_for_all_but_the_last_real_mma_group(sass, kernel):
    funcs, cur = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1) if kernel in m.group(1) else None
            if cur:
                funcs[cur] = []
        elif cur:
            funcs[cur].append(line)
    assert len(funcs) == 2, f"{kernel}<1> and <3> not both in the library: {list(funcs)}"
    for name, lines in funcs.items():
        lagged, last_hgmma = 0, None
        for line in lines:
            if "HGMMA" in line:
                last_hgmma = line
            if re.search(r"WARPGROUP\.DEPBAR\.LE gsb0, 0x1\b", line):
                lagged += 1
                assert last_hgmma is not None and "gdesc[URZ]" not in last_hgmma, \
                    f"{name}: wait_group 1 follows an empty dummy MMA group: {last_hgmma.strip()}"
        assert lagged > 0, f"{name}: no wgmma.wait_group 1 (every slot drained)"


@pytest.mark.parametrize("stages", [3, 4, 5, 6, 7, 8])
@pytest.mark.parametrize("gbufs", [2, 3, 4])
@pytest.mark.parametrize("kernel", ["k_wgrad_pl", "k_wgrad_tc"])
def test_wgrad_roles_with_lagged_release_are_sound(kernel, gbufs, stages):
    # two consumer warpgroups take every slot; k_wgrad_pl: Wu = the largest divisor of `stages` <= 7 unit producers and
    # Wg = the largest divisor of `gbufs` <= 8 - Wu gout producers
    Wu = ps.producer_choice(stages) if kernel == "k_wgrad_pl" else 1
    Wg = ps.gout_producer_choice(gbufs, Wu) if kernel == "k_wgrad_pl" else 1
    for nunits in (1, 2):
        res = {ps.sim(Wu, nunits, stages, 2, 7, seed, every=True, lag=True, gbufs=gbufs, joint=kernel == "k_wgrad_tc", Wg=Wg)
               for seed in range(6)}
        assert res == {"ok"}, (kernel, stages, gbufs, nunits, Wu, Wg, res)


@pytest.mark.gpu
@pytest.mark.parametrize("prec,tol", [("fp32", 2e-5), ("bf16", 2e-2)])
@pytest.mark.parametrize("cin", [64, 128])
@pytest.mark.parametrize("planes", [True, False])
def test_wgrad_192_columns_matches_fp64(planes, cin, prec, tol):
    """Cout = 192 runs units of 64 columns, two per pass, in column ranges r and (r + 1) % 3: a pass's gout tile holds
    two blocks that are not adjacent in gout (or one, in the last pass when the unit count is odd: Cin = 128)."""
    from pasco_b200 import build
    build.build()
    from pasco_b200 import ops
    g = torch.Generator().manual_seed(5)
    occ = torch.rand(48, 40, 16, generator=g) < 0.35
    c = torch.nonzero(occ).int()
    C = torch.cat([torch.zeros(c.shape[0], 1, dtype=torch.int32), c], 1).cuda()
    N = C.shape[0]
    assert N % 64 != 0
    table, _ = ops.hash_insert(C)
    nbr = ops.kernel_map_probe(C, table, 3, (1, 1, 1))
    F = torch.randn(N, cin, generator=g).cuda()
    G = torch.randn(N, 192, generator=g).cuda()
    ops.set_precision(prec)
    ops.use_planes(planes)
    try:
        assert ops.conv_path("wgrad", cin, 192, 27, nbr, N) == ("planes" if planes else "regs")
        dW = ops.conv_wgrad(F, G, nbr, 27, cin, 192)
    finally:
        ops.use_planes(True)
        ops.set_precision("fp32")
    Fd, Gd = F.double(), G.double()
    ref = torch.stack([Fd[nbr[k].long().clamp(min=0)].mul((nbr[k] >= 0).double()[:, None]).T @ Gd for k in range(27)])
    err = float((dW.double() - ref).abs().max() / ref.abs().max())
    assert err <= tol, f"wgrad error {err:.3e}"
