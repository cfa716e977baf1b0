"""Sparse convolutions on the tensor cores at every network width: Cin and Cout multiples of 16, Cout <= 512
(conv_tc.cu / wgrad_tc.cu channel rules, DESIGN.md §3.1-3.3).

CPU part : ops.conv_path picks a tensor-core path for every shape inside that contract and the CUDA-core kernels outside
           it; the width fixtures' parameter manifests equal PascoNet(f).reference_state_dict().
GPU part : forward, input gradient and weight gradient against the oracle at contractions that are not multiples of 64
           and outputs wider than 256 columns, on the plane- and the register-gather kernels, in fp32 and bf16 mode;
           split-K, the fused epilogue statistics, plane vs register gather bit for bit; PascoNet(f = 32 / 96) against
           golden vectors of the unmodified reference (tests/golden/make_golden_widths.py), and one training step at
           every width f = 16 … 128 without a CUDA-core convolution launch.

The ring depths the planners pick for these shapes stay inside the ranges the lag replays of tests/test_pipeline_lag.py
and tests/test_wgrad_pipeline.py cover (unit / A rings 3-8, B rings 2-3, gout rings 2-4, 1 or 2 units per row tile).
"""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import parity  # noqa: E402
from parity import TOL_BF16, TOL_TIGHT, relerr  # noqa: E402

MANIFEST = parity.manifest("net_cfg1_widths_manifest.json")


@pytest.fixture(scope="module")
def ME():
    return parity.engine()


# ------------------------------------------------------------------------------------------------
# CPU: path selection and manifests
# ------------------------------------------------------------------------------------------------
class _SplitKLib:
    """Stands in for the library's split-K planner: split when K >= 18 and the output has few rows."""

    @staticmethod
    def pasco_conv_splitk_workspace_bytes(K, n_out, c_out):
        return 4 * K * n_out * c_out if K >= 18 and n_out <= 8192 else 0


def test_conv_path_follows_the_channel_contract(monkeypatch):
    from pasco_b200 import ops
    monkeypatch.setattr(ops, "load", lambda: _SplitKLib)
    nbr = object()                                   # conv_path only asks whether a table exists
    inside = range(16, 513, 16)
    for ci in list(inside) + [1024]:
        for co in inside:
            assert ops.conv_path("fwd", ci, co, 27, nbr, 100_000) == "planes", (ci, co)
            assert ops.conv_path("dgrad", ci, co, 8, nbr, 100_000) == "planes", (ci, co)
            assert ops.conv_path("fwd", ci, co, 1, None, 100_000) == "regs", (ci, co)
            assert ops.conv_path("fwd", ci, co, 245, nbr, 4096) == "splitk", (ci, co)
            assert ops.conv_path("wgrad", ci, co, 27, nbr, 100_000) == "planes", (ci, co)
            assert ops.conv_path("wgrad", ci, co, 1, None, 100_000) == "regs", (ci, co)
    ops.use_planes(False)
    try:
        for ci, co in ((32, 32), (96, 384), (512, 512)):
            assert ops.conv_path("fwd", ci, co, 27, nbr, 100_000) == "regs"
            assert ops.conv_path("wgrad", ci, co, 27, nbr, 100_000) == "regs"
    finally:
        ops.use_planes(True)
    for ci, co in ((8, 64), (24, 64), (40, 32), (64, 8), (64, 24), (64, 520), (64, 528), (64, 1024), (0, 64)):
        for kind in ("fwd", "dgrad", "wgrad"):
            assert ops.conv_path(kind, ci, co, 27, nbr, 100_000) == "simt", (kind, ci, co)
    assert ops.conv_path("fwd", 64, 64, 1025, nbr, 100_000) == "simt"
    ops.force_simt(True)
    try:
        assert ops.conv_path("fwd", 32, 32, 27, nbr, 100_000) == "simt"
        assert ops.conv_path("wgrad", 384, 384, 27, nbr, 100_000) == "simt"
    finally:
        ops.force_simt(False)


@pytest.mark.parametrize("f", [32, 96])
def test_width_manifest_matches_pasconet_state_dict(f):
    mine = {k: list(v.shape) for k, v in parity.pasconet(f=f).reference_state_dict().items()}
    ref = MANIFEST["params"][str(f)]
    assert sorted(mine) == sorted(ref), (sorted(set(ref) - set(mine))[:5], sorted(set(mine) - set(ref))[:5])
    bad = [k for k in ref if mine[k] != ref[k]]
    assert not bad, bad[:5]


# ------------------------------------------------------------------------------------------------
# GPU: kernels against the oracle
# ------------------------------------------------------------------------------------------------
# (kind, Cin, Cout): contractions of 16 … 512 channels (forward: Cin, input gradient: Cout), outputs of 16 … 512 columns
CASES = [("k3", 16, 16), ("k3", 32, 32), ("k3", 48, 80), ("k3", 80, 48), ("k3", 96, 96), ("k3", 160, 160),
         ("k3", 32, 64), ("k3", 96, 192), ("k3", 384, 192), ("k3", 320, 320),
         ("down", 32, 64), ("down", 96, 192), ("down", 160, 320), ("down", 256, 512),
         ("up", 64, 32), ("up", 384, 192), ("up", 512, 384), ("up", 160, 80)]
BF16_CASES = [("k3", 32, 32), ("k3", 80, 48), ("down", 160, 320), ("up", 512, 384)]


def _widths_case(ME, kind, cin, cout, prec, planes, tol):
    from pasco_b200 import ops
    ops.set_precision(prec)
    ops.use_planes(planes)
    try:
        with parity.launches() as launches:
            e = parity.run_conv_case(ME, kind, cin, cout, tol)
    finally:
        ops.use_planes(True)
        ops.set_precision("fp32")
    kinds = {k for k, *_ in launches}
    assert kinds == {"fwd", "dgrad", "wgrad"}, launches
    want = "planes" if planes else "regs"      # forward / input gradient: or split-K (few tiles x 27 offsets)
    assert all(p == want or (k != "wgrad" and p == "splitk") for k, p, _, _ in launches), launches
    print(f"{prec} {'planes' if planes else 'regs'} {kind} {cin}->{cout}: fwd {e[0]:.2e} dgrad {e[1]:.2e} wgrad {e[2]:.2e}")


@pytest.mark.gpu
@pytest.mark.parametrize("planes", [True, False])
@pytest.mark.parametrize("kind,cin,cout", CASES)
def test_conv_widths_fp32_match_oracle(ME, kind, cin, cout, planes):
    _widths_case(ME, kind, cin, cout, "fp32", planes, TOL_TIGHT)


@pytest.mark.gpu
@pytest.mark.parametrize("planes", [True, False])
@pytest.mark.parametrize("kind,cin,cout", BF16_CASES)
def test_conv_widths_bf16_match_oracle(ME, kind, cin, cout, planes):
    _widths_case(ME, kind, cin, cout, "bf16", planes, TOL_BF16)


@pytest.mark.gpu
@pytest.mark.parametrize("cin,cout", [(384, 384), (96, 384), (32, 48)])
def test_conv_widths_split_k_match_fp64(cin, cout):
    """Box kernel (5, 5, 3) over 8 output tiles: the split-K kernels cover every column range of a 384-channel output
    and the zero-padded contraction of 96 and 32 channels; forward and input gradient against fp64, deterministic."""
    from pasco_b200 import ops
    ops.set_precision("fp32")
    g = torch.Generator().manual_seed(12)
    grid = torch.stack(torch.meshgrid(torch.arange(16), torch.arange(16), torch.arange(4), indexing="ij"), -1).view(-1, 3)
    C = torch.cat([torch.zeros(grid.shape[0], 1, dtype=torch.int64), grid], 1).int().cuda()
    N = C.shape[0]
    table, _ = ops.hash_insert(C)
    nbr = ops.kernel_map_box(C, table, (5, 5, 3), (1, 1, 1))
    K = nbr.shape[0]
    assert ops.conv_path("fwd", cin, cout, K, nbr, N) == "splitk" and ops.conv_path("dgrad", cout, cin, K, nbr, N) == "splitk"
    F = torch.randn(N, cin, generator=g).cuda()
    W = (torch.randn(K, cin, cout, generator=g) * 0.05).cuda()
    b = torch.randn(cout, generator=g).cuda()
    G = torch.randn(N, cout, generator=g).cuda()
    koff = [K - 1 - k for k in range(K)]
    with parity.launches() as launches:
        o_f = ops.conv_apply(F, W, nbr, N, False, None, b)
        o_g = ops.conv_apply(G, W, nbr, N, True, koff)
    assert [p for _, p, _, _ in launches] == ["splitk", "splitk"]
    Fd, Gd, Wd = F.double(), G.double(), W.double()
    ref_f = torch.zeros(N, cout, dtype=torch.float64, device="cuda") + b.double()
    ref_g = torch.zeros(N, cin, dtype=torch.float64, device="cuda")
    for k in range(K):
        src = nbr[k].long()
        ok = src >= 0
        ref_f[ok] += Fd[src[ok]] @ Wd[k]
        ref_g[ok] += Gd[src[ok]] @ Wd[koff[k]].t()
    assert relerr(o_f, ref_f) <= 1e-4 and relerr(o_g, ref_g) <= 1e-4, (relerr(o_f, ref_f), relerr(o_g, ref_g))
    assert torch.equal(ops.conv_apply(F, W, nbr, N, False, None, b), o_f)


def _probe_scene(seed, shape, p):
    from pasco_b200 import ops
    g = torch.Generator().manual_seed(seed)
    c = torch.nonzero(torch.rand(*shape, generator=g) < p).int()
    C = torch.cat([torch.zeros(c.shape[0], 1, dtype=torch.int32), c], 1).cuda()
    table, _ = ops.hash_insert(C)
    return g, C.shape[0], ops.kernel_map_probe(C, table, 3, (1, 1, 1))


@pytest.mark.gpu
@pytest.mark.parametrize("cin,cout,bias", [(32, 32, True), (48, 80, False), (96, 384, True)])
def test_conv_widths_epilogue_statistics(cin, cout, bias):
    """The fused BatchNorm statistics cover every column range: 32, 80 (16-column chunks) and 384 (three ranges)."""
    from pasco_b200 import ops
    ops.set_precision("fp32")
    g, N, nbr = _probe_scene(5, (48, 40, 16), 0.3)
    assert N >= 4096 and N % 128 != 0
    F = torch.randn(N, cin, generator=g).cuda()
    W = (torch.randn(27, cin, cout, generator=g) * 0.1).cuda()
    b = torch.randn(cout, generator=g).cuda() if bias else None
    ops.split_k(False)
    try:
        out = ops.conv_apply(F, W, nbr, N, False, None, b, want_stats=True)
        got = ops.take_pending_stats(out)
        assert got is not None
        assert relerr(got, ops.column_stats(out)) <= 1e-6
    finally:
        ops.split_k(True)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("cin,cout", [(32, 32), (384, 384), (48, 160)])
def test_conv_widths_plane_and_register_gather_are_bit_identical(prec, cin, cout):
    """Zero-fill copies (k_conv_pl) and zero stores (k_conv_tc) of the channels past Cin give the same operand tiles:
    forward with bias and statistics and input gradient bit for bit, the weight gradient to its summation order."""
    from pasco_b200 import ops
    ops.set_precision(prec)
    g, N, nbr = _probe_scene(4, (48, 40, 14), 0.35)
    F = torch.randn(N, cin, generator=g).cuda()
    G = torch.randn(N, cout, generator=g).cuda()
    W = (torch.randn(27, cin, cout, generator=g) * 0.05).cuda()
    b = torch.randn(cout, generator=g).cuda()
    koff = [26 - k for k in range(27)]
    res = []
    ops.split_k(False)
    try:
        for flag in (True, False):
            ops.use_planes(flag)
            pk = ops.PackedWeights()
            f = ops.conv_apply(F, W, nbr, N, False, None, b, packs=pk, want_stats=True)
            st = ops.take_pending_stats(f)
            d = ops.conv_apply(G, W, nbr, N, True, koff, packs=pk)
            w = ops.conv_wgrad(F, G, nbr, 27, cin, cout)
            res.append((f, st, d, w))
    finally:
        ops.use_planes(True)
        ops.split_k(True)
        ops.set_precision("fp32")
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][2], res[1][2])
    assert res[0][1] is not None and relerr(res[0][1], res[1][1]) <= 1e-12
    assert relerr(res[0][3], res[1][3]) <= 1e-5
    assert res[0][0].abs().sum() > 0 and res[0][3].abs().sum() > 0


# ------------------------------------------------------------------------------------------------
# GPU: the network at other widths
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("f", [32, 96])
def test_pasconet_width_matches_reference_golden(f):
    from pasco_b200 import ops
    ops.set_precision("fp32")
    net = parity.pasconet(f=f, recipe=True).cuda().train()
    with torch.no_grad(), parity.launches() as launches:
        out = parity.forward(net, parity.scene(MANIFEST))
    assert launches and not [x for x in launches if x[1] == "simt"], [x for x in launches if x[1] == "simt"][:5]
    report = parity.check_outputs(out, parity.fixture(f"net_cfg1_f{f}.npz"), MANIFEST, sums=True)
    print(f"PascoNet f={f} vs golden:", report)


@pytest.mark.gpu
@pytest.mark.parametrize("f", [16, 32, 48, 80, 96, 128])
def test_pasconet_width_training_step_runs_on_tensor_cores(f):
    """Forward + loss + backward + AdamW at width f: every convolution launch (forward, input and weight gradient,
    including the dense bottleneck) takes a tensor-core path, and every gradient is finite."""
    from pasco_b200 import ops
    from pasco_b200.losses import total_loss
    ops.set_precision("fp32")
    net = parity.pasconet(f=f).cuda().train()
    sc = parity.scene(MANIFEST)
    opt = torch.optim.AdamW(net.parameters(), lr=1e-4)
    with parity.launches() as launches:
        loss = total_loss(parity.forward(net, sc), sc, 20, net.class_frequencies)
        loss.backward()
    assert torch.isfinite(loss), loss
    simt = [x for x in launches if x[1] == "simt"]
    assert not simt, simt[:5]
    assert {k for k, *_ in launches} == {"fwd", "dgrad", "wgrad"}
    widths = {x[3] for x in launches if x[0] == "fwd"}
    assert {f, 2 * f, 4 * f} <= widths, sorted(widths)
    bad = [n for n, p in net.named_parameters() if p.grad is not None and not torch.isfinite(p.grad).all()]
    assert not bad, bad[:5]
    assert sum(p.grad is not None for p in net.parameters()) > 100
    opt.step()
