"""256-column weight-gradient units (`k_wgrad_n256`, DESIGN.md §3.2): one producer warpgroup, setmaxnreg, 32-row ring
slots and one m64n256k16 chain per k-step.

* The SASS of both precisions hands registers from the producers to the consumers, issues 64x256 MMAs and keeps one
  real MMA group in flight (no GPU needed).
* The lagged release is replayed under random schedules for every ring depth pair the planner can give this kernel, with
  its producer split: Wu = the largest divisor of `stages` <= 3 unit warps, Wg = the largest divisor of `gstages` <= 4 - Wu
  gout warps.
* On the GPU, dW at C_out = 256, 400 (last range zero past C_out) and 512 matches an fp64 reference, element by element
  relative to the sum of the absolute products it adds (the scale of both the bf16 split error and the fp32 summation
  error, which a bound relative to max |dW| does not follow as the row count grows).  At these shapes
  (169 row tiles) the 128-column grids take twice the waves of the 256-column ones on a 132-SM H100, so the launches run
  `k_wgrad_n256`."""
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


def test_wide_wgrad_kernels_move_registers_and_keep_one_mma_group_in_flight(sass):
    funcs, cur = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1) if "k_wgrad_n256" in m.group(1) else None
            if cur:
                funcs[cur] = []
        elif cur:
            funcs[cur].append(line)
    assert len(funcs) == 2, f"k_wgrad_n256<1> and <3> not both in the library: {list(funcs)}"
    for name, lines in funcs.items():
        text = "\n".join(lines)
        assert "USETMAXREG.DEALLOC" in text and "USETMAXREG.TRY_ALLOC" in text, f"{name}: no setmaxnreg"
        assert "HGMMA.64x256x16" in text, f"{name}: no m64n256k16 MMA"
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
def test_wide_wgrad_roles_with_lagged_release_are_sound(gbufs, stages):
    Wu = ps.producer_choice(stages, max_producers=3)
    Wg = ps.gout_producer_choice(gbufs, Wu, warps=4)
    res = {ps.sim(Wu, 1, stages, 2, 9, seed, every=True, lag=True, gbufs=gbufs, Wg=Wg) for seed in range(8)}
    assert res == {"ok"}, (stages, gbufs, Wu, Wg, res)


@pytest.mark.gpu
@pytest.mark.parametrize("prec,tol", [("fp32", 2e-5), ("bf16", 2e-2)])
@pytest.mark.parametrize("cin,cout", [(256, 256), (256, 400), (128, 512)])
def test_wide_wgrad_matches_fp64(cin, cout, prec, tol):
    from pasco_b200 import build
    build.build()
    from pasco_b200 import ops
    g = torch.Generator().manual_seed(7)
    occ = torch.rand(48, 40, 16, generator=g) < 0.35
    c = torch.nonzero(occ).int()
    C = torch.cat([torch.zeros(c.shape[0], 1, dtype=torch.int32), c], 1).cuda()
    N = C.shape[0]
    assert N % 64 > 32          # the last row tile's second 32-row slot is ragged
    table, _ = ops.hash_insert(C)
    nbr = ops.kernel_map_probe(C, table, 3, (1, 1, 1))
    F = torch.randn(N, cin, generator=g).cuda()
    G = torch.randn(N, cout, generator=g).cuda()
    ops.set_precision(prec)
    try:
        assert ops.conv_path("wgrad", cin, cout, 27, nbr, N) == "planes"
        dW = ops.conv_wgrad(F, G, nbr, 27, cin, cout)
        again = ops.conv_wgrad(F, G, nbr, 27, cin, cout)
    finally:
        ops.set_precision("fp32")
    assert torch.equal(dW, again)
    Fd, Gd = F.double(), G.double()
    A = [Fd[nbr[k].long().clamp(min=0)].mul((nbr[k] >= 0).double()[:, None]) for k in range(27)]
    ref = torch.stack([a.T @ Gd for a in A])
    scale = torch.stack([a.abs().T @ Gd.abs() for a in A])
    err = float(((dW.double() - ref).abs() / scale.clamp(min=1e-300)).max())
    print(f"{prec} {cin}->{cout}: error {err:.2e} of the absolute sums, "
          f"{float((dW.double() - ref).abs().max() / ref.abs().max()):.2e} of max |dW|")
    assert err <= tol, f"wgrad error {err:.3e} of the absolute sums"
