"""Parity of the CUDA path (through the C-ABI) against the CPU oracle on the same seeded inputs.

Integer work (coordinate maps, kernel maps) must match bit-exactly after canonicalisation
(rows sorted by (b,x,y,z); kernel maps compared as sets of (k, in_coord, out_coord) triples —
SURVEY.md §8c item 3).  fp32 features: max-abs-normalised error ≤ 1e-3 (north_star), in practice
~1e-5 for the bf16x3 path and exactly-rounded fp32 for the CUDA-core path.
"""
import os
import sys

import pytest
import torch

import me_oracle as OR

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import parity  # noqa: E402
from parity import (TOL_BF16, TOL_FP32, TOL_TIGHT, assert_same_sparse, canon, conv_pair, relerr,  # noqa: E402
                    run_conv_case, sparse_scene)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ME():
    return parity.engine()


def triples(nbr, in_c, out_c):
    """Canonical set of (k, in_key, out_key) triples of a neighbour table."""
    nbr = nbr.detach().cpu().long()
    ik, ok = OR.pack_keys(in_c.detach().cpu()), OR.pack_keys(out_c.detach().cpu())
    k, o = torch.nonzero(nbr >= 0, as_tuple=True)
    t = torch.stack([k, ik[nbr[k, o]], ok[o]], 1)
    return sorted(map(tuple, t.tolist()))


# ------------------------------------------------------------------------------------------------
# integer parity
# ------------------------------------------------------------------------------------------------
def test_insert_dedups_first_wins_and_keeps_order(ME):
    C, F = sparse_scene(p=0.2, C=8, lo=(-8, 4, -2))
    C2 = torch.cat([C, C[:50]], 0)
    F2 = torch.cat([F, F[:50] + 100.0], 0)
    ref = OR.SparseTensor(F2, C2)
    got = ME.SparseTensor(F2.cuda(), C2.cuda())
    assert torch.equal(got.C.cpu(), ref.C) and torch.equal(got.F.cpu(), ref.F)


@pytest.mark.parametrize("lo", [(0, 0, 0), (-16, -8, -4)])
def test_kernel_map_k3_bit_exact(ME, lo):
    C, F = sparse_scene(C=8, batch=2, lo=lo)
    ref = OR.SparseTensor(F, C)
    got = ME.SparseTensor(F.cuda(), C.cuda())
    rk = ref.coordinate_manager.kernel_map(ref.coordinate_map_key, ref.coordinate_map_key, 3)
    gk = got.coordinate_manager.kernel_map(got.coordinate_map_key, got.coordinate_map_key, 3, 1, 1, False)
    assert gk.nbr.shape == rk.shape
    assert triples(gk.nbr, got.C, got.C) == triples(rk, ref.C, ref.C)
    nbr_t, koff = gk.transposed()
    assert koff == [26 - k for k in range(27)]


@pytest.mark.parametrize("lo", [(0, 0, 0), (-16, -8, -4)])
def test_stride_map_and_down_kernel_map_bit_exact(ME, lo):
    C, F = sparse_scene(C=8, batch=2, lo=lo)
    ref = OR.SparseTensor(F, C)
    got = ME.SparseTensor(F.cuda(), C.cuda())
    rcm, gcm = ref.coordinate_manager, got.coordinate_manager
    rkey, gkey = rcm.stride(ref.coordinate_map_key, 2), gcm.stride(got.coordinate_map_key, 2)
    assert torch.equal(canon(gcm.get_coordinates(gkey))[0], canon(rcm.get_coordinates(rkey))[0])
    rk = rcm.kernel_map(ref.coordinate_map_key, rkey, 2)
    gk = gcm.kernel_map(got.coordinate_map_key, gkey, 2, 2, 1, False)
    assert triples(gk.nbr, got.C, gcm.get_coordinates(gkey)) == triples(rk, ref.C, rcm.get_coordinates(rkey))
    nbr_t, _ = gk.transposed()          # table over children: exactly one parent each
    assert int((nbr_t >= 0).sum()) == C.shape[0]


def test_generative_map_union_and_prune_bit_exact(ME):
    C, F = sparse_scene(shape=(6, 5, 4), p=0.5, C=8, stride=2, lo=(-4, 0, 2))
    ref = OR.SparseTensor(F, C, tensor_stride=2)
    got = ME.SparseTensor(F.cuda(), C.cuda(), tensor_stride=2)
    rkey = ref.coordinate_manager.generate(ref.coordinate_map_key, 2, 2)
    gkey = got.coordinate_manager.generate(got.coordinate_map_key, 2, 2)
    rc, gc = ref.coordinate_manager.get_coordinates(rkey), got.coordinate_manager.get_coordinates(gkey)
    assert torch.equal(canon(gc)[0], canon(rc)[0]) and gkey.tensor_stride == (1, 1, 1)
    # union of two partially overlapping sets inside one manager
    C2, F2 = sparse_scene(shape=(12, 10, 8), p=0.3, C=8, seed=5, lo=(-4, 0, 2))
    ra = OR.SparseTensor(torch.ones(rc.shape[0], 8), coordinate_map_key=rkey, coordinate_manager=ref.coordinate_manager)
    rb = OR.SparseTensor(F2, C2, coordinate_manager=ref.coordinate_manager)
    ga = ME.SparseTensor(torch.ones(gc.shape[0], 8).cuda(), coordinate_map_key=gkey,
                         coordinate_manager=got.coordinate_manager)
    gb = ME.SparseTensor(F2.cuda(), C2.cuda(), coordinate_manager=got.coordinate_manager)
    assert_same_sparse(ga + gb, ra + rb, 0.0)
    # prune keeps order
    m = torch.rand(C2.shape[0], generator=torch.Generator().manual_seed(3)) < 0.4
    rp, gp = OR.MinkowskiPruning()(rb, m), ME.MinkowskiPruning()(gb, m.cuda())
    assert torch.equal(gp.C.cpu(), rp.C) and torch.equal(gp.F.cpu(), rp.F)
    assert ME.MinkowskiPruning()(gb, torch.zeros_like(m).cuda()).F.shape == (0, 8)
    with pytest.raises(RuntimeError):
        ME.MinkowskiPruning()(gb, m[:-1].cuda())


def test_dense_and_to_sparse_match(ME):
    C, F = sparse_scene(shape=(9, 7, 5), p=0.4, C=6, batch=2, lo=(-4, 0, 2))
    F[5] = 0
    ref, got = OR.SparseTensor(F, C), ME.SparseTensor(F.cuda(), C.cuda())
    mn = torch.IntTensor([-4, 0, 2])
    rd, gd = ref.dense(min_coordinate=mn)[0], got.dense(min_coordinate=mn)[0]
    assert rd.shape == gd.shape and torch.equal(gd.cpu(), rd)
    rs, gs = OR.to_sparse(rd), ME.to_sparse(gd)
    assert torch.equal(gs.C.cpu(), rs.C) and torch.equal(gs.F.cpu(), rs.F)
    with pytest.raises(ValueError):
        got.dense()
    shp = torch.Size([2, 6, 12, 8, 6])
    assert torch.equal(got.dense(shp, min_coordinate=mn)[0].cpu(), ref.dense(shp, min_coordinate=mn)[0])


# ------------------------------------------------------------------------------------------------
# convolution parity (forward + both gradients), tensor-core and CUDA-core paths
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,cin,cout", [("k3", 64, 64), ("k3", 128, 128), ("k3", 256, 256), ("down", 64, 128),
                                           ("down", 128, 256), ("up", 256, 128), ("up", 128, 64), ("k3", 64, 128)])
def test_conv_tensor_core_fp32_mode(ME, kind, cin, cout):
    from pasco_b200 import ops
    ops.set_precision("fp32")
    ops.force_simt(False)
    e = run_conv_case(ME, kind, cin, cout, TOL_TIGHT, bias=(kind == "k3" and cin == 64 and cout == 64))
    print(f"bf16x3 {kind} {cin}->{cout}: fwd {e[0]:.2e} dgrad {e[1]:.2e} wgrad {e[2]:.2e}")


@pytest.mark.parametrize("kind,cin,cout", [("k3", 64, 64), ("down", 64, 128), ("up", 128, 64)])
def test_conv_tensor_core_bf16_mode(ME, kind, cin, cout):
    from pasco_b200 import ops
    ops.set_precision("bf16")
    try:
        e = run_conv_case(ME, kind, cin, cout, TOL_BF16)
        print(f"bf16 {kind} {cin}->{cout}: fwd {e[0]:.2e} dgrad {e[1]:.2e} wgrad {e[2]:.2e}")
    finally:
        ops.set_precision("fp32")


@pytest.mark.parametrize("kind,cin,cout", [("k3", 64, 64), ("k3", 24, 40), ("down", 16, 24), ("up", 24, 8)])
def test_conv_cuda_core_path(ME, kind, cin, cout):
    from pasco_b200 import ops
    ops.force_simt(True)
    try:
        e = run_conv_case(ME, kind, cin, cout, TOL_TIGHT, shape=(12, 10, 8))
    finally:
        ops.force_simt(False)


@pytest.mark.parametrize("kind,cin,cout", [("k3", 64, 64), ("k3", 128, 128), ("k3", 256, 256), ("down", 64, 128),
                                           ("up", 128, 64), ("k3", 64, 128)])
def test_conv_register_gather_path(ME, kind, cin, cout):
    """The round-1 kernels (k_conv_tc / k_wgrad_tc: fp32 rows gathered through registers, converted per offset) stay
    available as ops.use_planes(False); the default since round 2 is the plane-gather path the tests above ran."""
    from pasco_b200 import ops
    ops.set_precision("fp32")
    ops.use_planes(False)
    try:
        run_conv_case(ME, kind, cin, cout, TOL_TIGHT, bias=(cin == 64 and cout == 64))
    finally:
        ops.use_planes(True)


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("cin,cout", [(64, 64), (128, 64), (256, 256)])
def test_conv_plane_and_register_gather_are_bit_identical(prec, cin, cout):
    """Same operand split (x = hi + lo done once per tensor vs once per gathered copy), same MMA order and epilogue →
    k_conv_pl and k_conv_tc must agree bit for bit: forward with bias + fused statistics, input gradient with mirrored
    offsets, ragged last tile, ~40 % missing neighbours (zero-fill copies)."""
    from pasco_b200 import ops
    ops.set_precision(prec)
    g = torch.Generator().manual_seed(4)
    occ = torch.rand(48, 40, 14, generator=g) < 0.35
    c = torch.nonzero(occ).int()
    C = torch.cat([torch.zeros(c.shape[0], 1, dtype=torch.int32), c], 1).cuda()
    N = C.shape[0]
    assert N % 128 != 0 and N > 4096
    table, _ = ops.hash_insert(C)
    nbr = ops.kernel_map_probe(C, table, 3, (1, 1, 1))
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
    assert relerr(res[0][3], res[1][3]) <= 1e-5          # dW: the two kernels sum in different orders
    assert res[0][0].abs().sum() > 0


@pytest.mark.parametrize("cin,cout,bias", [(64, 64, False), (64, 128, True), (128, 256, False), (64, 48, True)])
def test_conv_epilogue_statistics(cin, cout, bias):
    """Fused BatchNorm statistics: the conv epilogue's column sums / sums of squares of its output (incl. bias, a ragged
    last tile and the 16-column tail of Cout = 48) equal a separate pass over the stored output; they are handed to the
    next BatchNormAct only for the untouched tensor."""
    from pasco_b200 import ops
    ops.set_precision("fp32")
    g = torch.Generator().manual_seed(5)
    occ = torch.rand(48, 40, 16, generator=g) < 0.3
    c = torch.nonzero(occ).int()
    C = torch.cat([torch.zeros(c.shape[0], 1, dtype=torch.int32), c], 1).cuda()
    N = C.shape[0]
    assert N >= 4096 and N % 128 != 0
    table, _ = ops.hash_insert(C)
    nbr = ops.kernel_map_probe(C, table, 3, (1, 1, 1))
    F = torch.randn(N, cin, generator=g).cuda()
    W = (torch.randn(27, cin, cout, generator=g) * 0.1).cuda()
    b = torch.randn(cout, generator=g).cuda() if bias else None
    ops.split_k(False)            # 72 tiles x 27 offsets would otherwise take the split-K path (no fused statistics there)
    try:
        out = ops.conv_apply(F, W, nbr, N, False, None, b, want_stats=True)
        ref = ops.column_stats(out)
        got = ops.take_pending_stats(out)
        assert got is not None and ops.take_pending_stats(out) is None          # consumed once
        assert relerr(got, ref) <= 1e-6
        out2 = ops.conv_apply(F, W, nbr, N, False, None, b, want_stats=True)
        out2.add_(1.0)                                                           # in-place change → statistics are stale
        assert ops.take_pending_stats(out2) is None
    finally:
        ops.split_k(True)


@pytest.mark.parametrize("kernel,cin,cout,bias", [((7, 7, 5), 64, 64, True), ((5, 5, 3), 128, 128, False), ((3, 3, 3), 64, 128, True)])
def test_conv_split_k_matches_unsplit(kernel, cin, cout, bias):
    """Few output tiles x many offsets (the dense-bottleneck shape) run as (tile, offset-range) work items with a
    deterministic reduction; result = the one-CTA-per-tile kernel up to the fp32 accumulation order of K*Cin (up to 15,680)
    products per output — both are compared with an fp64 evaluation of the same contraction, incl. mirrored offsets."""
    from pasco_b200 import ops
    ops.set_precision("fp32")
    g = torch.Generator().manual_seed(11)
    X, Y, Z = 16, 16, 4
    grid = torch.stack(torch.meshgrid(torch.arange(X), torch.arange(Y), torch.arange(Z), indexing="ij"), -1).view(-1, 3)
    C = torch.cat([torch.zeros(grid.shape[0], 1, dtype=torch.int64), grid], 1).int().cuda()
    N = C.shape[0]
    table, _ = ops.hash_insert(C)
    nbr = ops.kernel_map_box(C, table, kernel, (1, 1, 1))
    K = nbr.shape[0]
    assert ops.load().pasco_conv_splitk_workspace_bytes(K, N, cout) > 0
    F = torch.randn(N, cin, generator=g).cuda()
    W = (torch.randn(K, cin, cout, generator=g) * 0.05).cuda()
    b = torch.randn(cout, generator=g).cuda() if bias else None
    G = torch.randn(N, cout, generator=g).cuda()
    koff = [K - 1 - k for k in range(K)]
    outs = []
    try:
        for flag in (True, False):
            ops.split_k(flag)
            outs.append((ops.conv_apply(F, W, nbr, N, False, None, b), ops.conv_apply(G, W, nbr, N, True, koff)))
    finally:
        ops.split_k(True)
    Fd, Gd, Wd = F.double(), G.double(), W.double()
    ref_f = torch.zeros(N, cout, dtype=torch.float64, device="cuda") + (b.double() if bias else 0.0)
    ref_g = torch.zeros(N, cin, dtype=torch.float64, device="cuda")
    for k in range(K):
        src = nbr[k].long()
        ok = src >= 0
        ref_f[ok] += Fd[src[ok]] @ Wd[k]
        ref_g[ok] += Gd[src[ok]] @ Wd[koff[k]].t()
    # 245 x 64 products accumulate in fp32 register accumulators: 1e-4 of the output range (the parity bound is 1e-3)
    for o_f, o_g in outs:
        assert relerr(o_f, ref_f) <= 1e-4 and relerr(o_g, ref_g) <= 1e-4
    assert relerr(outs[0][0], outs[1][0]) <= 2e-4 and relerr(outs[0][1], outs[1][1]) <= 2e-4
    again = ops.conv_apply(F, W, nbr, N, False, None, b)
    assert torch.equal(again, outs[0][0])                       # deterministic


def test_conv_many_tiles_per_cta(ME):
    """~59k voxels: every persistent CTA walks several 128-row tiles (and several 64-row wgrad tiles
    accumulating in registers), unlike the small cases above."""
    from pasco_b200 import ops
    ops.set_precision("fp32")
    e = run_conv_case(ME, "k3", 64, 64, TOL_TIGHT, shape=(64, 64, 32), p=0.225)
    print(f"bf16x3 k3 64->64 @59k rows: fwd {e[0]:.2e} dgrad {e[1]:.2e} wgrad {e[2]:.2e}")


def test_conv_benchmark_scale_rows_match_fp64():
    """The largest layer shape of the benchmark (≈1 M rows, C = 64, K = 27, ~17 M pairs): forward, input gradient and
    weight gradient of the plane-gather kernels against an fp64 evaluation on a 1/64 row subsample (forward / dgrad) and
    the full fp64 contraction for two offsets (wgrad) — every persistent CTA walks ~56 tile groups here."""
    from pasco_b200 import ops
    ops.set_precision("fp32")
    g = torch.Generator().manual_seed(9)
    occ = torch.rand(256, 256, 32, generator=g) < 0.5
    c = torch.nonzero(occ).int()
    C = torch.cat([torch.zeros(c.shape[0], 1, dtype=torch.int32), c], 1).cuda()
    N = C.shape[0]
    assert N > 1_000_000
    table, _ = ops.hash_insert(C)
    nbr = ops.kernel_map_probe(C, table, 3, (1, 1, 1))
    F = torch.randn(N, 64, generator=g).cuda()
    G = torch.randn(N, 64, generator=g).cuda()
    W = (torch.randn(27, 64, 64, generator=g) * 0.05).cuda()
    koff = [26 - k for k in range(27)]
    out = ops.conv_apply(F, W, nbr, N, False, None)
    din = ops.conv_apply(G, W, nbr, N, True, koff)
    dW = ops.conv_wgrad(F, G, nbr, 27, 64, 64)
    rows = torch.arange(0, N, 64, device="cuda")
    ref_f = torch.zeros(rows.numel(), 64, dtype=torch.float64, device="cuda")
    ref_d = torch.zeros_like(ref_f)
    Fd, Gd, Wd = F.double(), G.double(), W.double()
    for k in range(27):
        src = nbr[k][rows].long()
        ok = src >= 0
        ref_f[ok] += Fd[src[ok]] @ Wd[k]
        ref_d[ok] += Gd[src[ok]] @ Wd[koff[k]].t()
    assert relerr(out[rows], ref_f) <= TOL_TIGHT and relerr(din[rows], ref_d) <= TOL_TIGHT
    for k in (0, 13):
        src = nbr[k].long()
        ok = src >= 0
        ref_w = Fd[src[ok]].t() @ Gd[ok]
        assert relerr(dW[k], ref_w) <= 1e-4, k        # ~650 k rows accumulate per entry in fp32 (registers + the CTA partials summed in order)


def test_conv_tile_tail_and_single_voxel(ME):
    """n_out not a multiple of the 128-row tile, and a 1-voxel tensor."""
    from pasco_b200 import ops
    ops.set_precision("fp32")
    for shape, p in (((7, 6, 5), 0.63), ((1, 1, 1), 1.1)):
        C, F = sparse_scene(shape=shape, p=p, C=64)
        rconv, gconv = conv_pair(ME, "k3", 64, 64)
        assert_same_sparse(gconv(ME.SparseTensor(F.cuda(), C.cuda())), rconv(OR.SparseTensor(F, C)), TOL_TIGHT)


def test_conv_full_grid_matches_dense_conv3d(ME):
    """Independent of the oracle: on a fully occupied grid the sparse conv IS F.conv3d(padding=1)."""
    import torch.nn.functional as Fn
    X, Y, Z, Cc = 10, 9, 8, 64
    g = torch.Generator().manual_seed(1)
    dense = torch.randn(1, Cc, X, Y, Z, generator=g)
    idx = torch.nonzero(torch.ones(X, Y, Z)).int()
    C = OR.utils.batched_coordinates([idx])
    F = dense[0, :, idx[:, 0].long(), idx[:, 1].long(), idx[:, 2].long()].t().contiguous()
    conv = ME.MinkowskiConvolution(Cc, Cc, kernel_size=3, dimension=3).cuda()
    y = conv(ME.SparseTensor(F.cuda(), C.cuda()))
    w = conv.kernel.detach().cpu().view(3, 3, 3, Cc, Cc).permute(4, 3, 2, 1, 0).contiguous()
    ref = Fn.conv3d(dense.double(), w.double(), padding=1)[0]
    c = y.C.cpu().long()
    assert relerr(y.F, ref[:, c[:, 1], c[:, 2], c[:, 3]].t()) <= TOL_TIGHT


# ------------------------------------------------------------------------------------------------
# pooling / scatter-max / batch-norm
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("s", [2, 4])
def test_maxpool_matches(ME, s):
    C, F = sparse_scene(shape=(16, 12, 8), p=0.4, C=10, batch=2, lo=(-8, 0, 4))
    ref = OR.MinkowskiMaxPooling(kernel_size=s, stride=s, dimension=3)(OR.SparseTensor(F, C))
    got = ME.MinkowskiMaxPooling(kernel_size=s, stride=s, dimension=3)(ME.SparseTensor(F.cuda(), C.cuda()))
    assert_same_sparse(got, ref, 0.0)


def test_scatter_max_matches(ME):
    g = torch.Generator().manual_seed(0)
    src = torch.randn(5000, 64, generator=g)
    idx = torch.randint(0, 700, (5000,), generator=g)
    idx[idx == 13] = 14                                       # an empty segment
    rv, ra = OR.scatter_max(src, idx, dim=0)
    src_g = src.clone().cuda().requires_grad_(True)
    gv, ga = ME.scatter_max(src_g, idx.cuda(), dim=0)
    assert torch.equal(gv.cpu(), rv) and torch.equal(ga.cpu(), ra)
    assert float(gv[13].abs().sum()) == 0.0
    src_r = src.clone().requires_grad_(True)
    OR.scatter_max(src_r, idx, dim=0)[0].sum().backward()
    gv.sum().backward()
    assert torch.equal(src_g.grad.cpu(), src_r.grad)


@pytest.mark.parametrize("C,act", [(64, 1), (67, 0), (128, 2), (20, 1)])
def test_fused_batchnorm_act_forward_backward(ME, C, act):
    from pasco_b200 import ops
    g = torch.Generator().manual_seed(0)
    x = (torch.randn(3001, C, generator=g) * 2 + 0.5)
    gamma, beta = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g)
    up = torch.randn(3001, C, generator=g)
    xr = x.clone().double().requires_grad_(True)
    gr, br = gamma.clone().double().requires_grad_(True), beta.clone().double().requires_grad_(True)
    z = torch.nn.functional.batch_norm(xr, None, None, gr, br, True, 0.1, 1e-5)
    yr = [z, torch.relu(z), torch.nn.functional.leaky_relu(z, 0.01)][act]
    (yr * up.double()).sum().backward()
    xg = x.clone().cuda().requires_grad_(True)
    gg, bg = gamma.clone().cuda().requires_grad_(True), beta.clone().cuda().requires_grad_(True)
    rm, rv = torch.zeros(C, device="cuda"), torch.ones(C, device="cuda")
    yg = ops.BatchNormAct.apply(xg, gg, bg, 1e-5, act, None, rm, rv, 0.1)
    (yg * up.cuda()).sum().backward()
    assert relerr(yg, yr) <= TOL_TIGHT
    assert relerr(xg.grad, xr.grad) <= 1e-4 and relerr(gg.grad, gr.grad) <= 1e-4 and relerr(bg.grad, br.grad) <= 1e-4
    # running statistics as torch.nn.BatchNorm1d keeps them (momentum 0.1, unbiased variance)
    assert relerr(rm, 0.1 * x.double().mean(0)) <= 1e-5
    assert relerr(rv, 0.9 + 0.1 * x.double().var(0, unbiased=True)) <= 1e-5


# ------------------------------------------------------------------------------------------------
# dense Linear layers on the tensor-core conv kernel
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,cin,cout,bias", [(5000, 64, 384, True), (6000, 384, 384, True), (4500, 384, 128, False),
                                              (4100, 128, 64, True)])
def test_linear_tensor_core_matches_fp64(ME, n, cin, cout, bias):
    from pasco_b200 import ops
    ops.set_precision("fp32")
    g = torch.Generator().manual_seed(n)
    x, w = torch.randn(n, cin, generator=g), torch.randn(cout, cin, generator=g) / cin ** 0.5
    b = torch.randn(cout, generator=g) if bias else None
    up = torch.randn(n, cout, generator=g)
    xr, wr = x.double().requires_grad_(True), w.double().requires_grad_(True)
    br = b.double().requires_grad_(True) if bias else None
    (torch.nn.functional.linear(xr, wr, br) * up.double()).sum().backward()
    xg, wg = x.cuda().requires_grad_(True), w.cuda().requires_grad_(True)
    bg = b.cuda().requires_grad_(True) if bias else None
    y = ops.linear(xg, wg, bg)
    assert y.grad_fn.__class__.__name__ == "LinearTCBackward"
    (y * up.cuda()).sum().backward()
    e = [relerr(y, torch.nn.functional.linear(xr, wr, br)), relerr(xg.grad, xr.grad), relerr(wg.grad, wr.grad)]
    if bias:
        e.append(relerr(bg.grad, br.grad))
    print(f"linear {n}x{cin}->{cout}: " + " ".join(f"{v:.1e}" for v in e))
    assert max(e) <= TOL_TIGHT


# ------------------------------------------------------------------------------------------------
# masked cross-attention kernel
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("P,Q,H,D,masked", [
    (3000, 100, 8, 48, True), (64, 100, 8, 48, True), (37, 5, 8, 48, False), (20011, 100, 8, 48, True),
    (3000, 128, 6, 64, True),          # no query or head-dim padding
    (1000, 100, 4, 20, True),          # a head that ends inside a 16-byte chunk of the bf16 operand tiles
])
def test_masked_cross_attention_matches_reference(ME, P, Q, H, D, masked):
    from pasco_b200 import ops
    g = torch.Generator().manual_seed(P)
    q, k, v = (torch.randn(n, H * D, generator=g) for n in (Q, P, P))
    mask = None
    if masked:
        mask = torch.rand(Q, P, generator=g) < 0.6
        mask[3] = True
        mask[3, P // 2] = False                         # a row with a single visible key
        mask[mask.all(1)] = False
    up = torch.randn(Q, H * D, generator=g)

    def ref(q, k, v):
        hv = lambda t: t.view(t.shape[0], H, D).transpose(0, 1)              # noqa: E731
        s = torch.bmm(hv(q) * D ** -0.5, hv(k).transpose(1, 2))
        if mask is not None:
            s = s.masked_fill(mask.unsqueeze(0), float("-inf"))
        return torch.bmm(torch.softmax(s, -1), hv(v)).transpose(0, 1).reshape(Q, H * D)

    qr, kr, vr = (t.clone().double().requires_grad_(True) for t in (q, k, v))
    yr = ref(qr, kr, vr)
    (yr * up.double()).sum().backward()
    qg, kg, vg = (t.clone().cuda().requires_grad_(True) for t in (q, k, v))
    yg = ops.MaskedCrossAttention.apply(qg, kg, vg, mask.cuda() if mask is not None else None, H)
    (yg * up.cuda()).sum().backward()
    e = relerr(yg, yr)
    eg = max(relerr(qg.grad, qr.grad), relerr(kg.grad, kr.grad), relerr(vg.grad, vr.grad))
    print(f"xattn P={P} Q={Q} H={H} D={D}: fwd {e:.2e} grads {eg:.2e}")
    assert e <= 1e-4 and eg <= 5e-4      # backward = fp32 library GEMMs against an fp64 reference


# ------------------------------------------------------------------------------------------------
# a residual U-Net slice written against the ME API (what pasco/maskpls/mink.py composes)
# ------------------------------------------------------------------------------------------------
def _mini_net(M):
    import torch.nn as nn

    class Res(nn.Module):
        def __init__(self, c):
            super().__init__()
            self.net = nn.Sequential(M.MinkowskiBatchNorm(c), M.MinkowskiReLU(inplace=True),
                                     M.MinkowskiConvolution(c, c, kernel_size=3, dimension=3),
                                     M.MinkowskiBatchNorm(c), M.MinkowskiReLU(inplace=True),
                                     M.MinkowskiConvolution(c, c, kernel_size=3, dimension=3))
            self.relu = M.MinkowskiReLU(inplace=True)

        def forward(self, x):
            return self.relu(x + self.net(x))

    class Net(nn.Module):
        def __init__(self):
            super().__init__()
            self.stem = M.MinkowskiConvolution(16, 64, kernel_size=1, dimension=3)
            self.r1 = Res(64)
            self.down = nn.Sequential(M.MinkowskiConvolution(64, 128, kernel_size=2, stride=2, dimension=3),
                                      M.MinkowskiBatchNorm(128), M.MinkowskiLeakyReLU(inplace=True))
            self.r2 = Res(128)
            self.up = nn.Sequential(M.MinkowskiConvolutionTranspose(128, 64, kernel_size=2, stride=2, dimension=3,
                                                                    expand_coordinates=True),
                                    M.MinkowskiBatchNorm(64), M.MinkowskiLeakyReLU(inplace=True))
            self.r3 = Res(64)
            self.head = M.MinkowskiConvolution(64, 20, kernel_size=1, bias=True, dimension=3)
            self.prune = M.MinkowskiPruning()

        def forward(self, x):
            s1 = self.r1(self.stem(x))
            s2 = self.r2(self.down(s1))
            u = self.up(s2)
            keep = (u.C[:, 1] >= 0) & (u.C[:, 1] < 20) & (u.C[:, 2] >= 0) & (u.C[:, 3] >= 0)
            u = self.prune(u, keep)
            return self.head(self.r3(u + s1))
    return Net()


@pytest.mark.parametrize("simt", [None, "all", "fwd", "dgrad", "wgrad"])
def test_unet_slice_forward_backward_matches_oracle(ME, simt):
    from pasco_b200 import ops
    ops.set_precision("fp32")
    ops.force_simt(simt is not None, None if simt in (None, "all") else [simt])
    torch.manual_seed(0)
    rnet = _mini_net(OR)
    gnet = _mini_net(ME)
    gnet.load_state_dict(rnet.state_dict())
    gnet.cuda()
    C, F = sparse_scene(shape=(20, 16, 8), p=0.25, C=16, batch=1)
    ry = rnet(OR.SparseTensor(F, C))
    gy = gnet(ME.SparseTensor(F.cuda(), C.cuda()))
    e = assert_same_sparse(gy, ry, TOL_FP32)
    (ry.F ** 2).mean().backward()
    (gy.F ** 2).mean().backward()
    ops.force_simt(False)
    # Gradients flow through ReLU masks: a forward difference of 1e-5 flips the sign of a handful of
    # pre-activations (out of ~1e5), each flip moving a parameter gradient by ~1/sqrt(rows*K) of its
    # max — so judge gradients in the relative L2 norm (robust to single flips), max-norm only loosely.
    def l2(a, b):
        a, b = a.detach().double().cpu(), b.detach().double().cpu()
        return float((a - b).norm() / b.norm().clamp(min=1e-30))
    errs = {n: (l2(pg.grad, pr.grad), relerr(pg.grad, pr.grad))
            for (n, pr), (_, pg) in zip(rnet.named_parameters(), gnet.named_parameters())}
    worst = max(errs, key=lambda n: errs[n][0])
    print(f"unet slice (simt={simt}): fwd {e:.2e}; worst param-grad rel-L2 {errs[worst][0]:.1e} ({worst}), "
          f"worst max-norm {max(v[1] for v in errs.values()):.1e}")
    # forward on the CUDA-core path (identical ReLU masks): the tensor-core dgrad/wgrad must agree to 1e-3;
    # forward on the tensor-core path: a couple of flipped masks in this 2.3k-voxel net move gradients by ~1/sqrt(rows*K)
    tol = 1e-3 if simt in ("all", "fwd") else 2e-2
    assert errs[worst][0] <= tol, worst
    assert max(v[1] for v in errs.values()) <= 5 * tol
