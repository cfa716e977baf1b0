"""The trunk hook (pasco_b200/hooks.py install(trunk=True)): the unmodified reference's CylinderFeat.forward,
Augmenter.merge and UNet3DV2.dense_bottleneck on csrc/voxel.cu and net3d's grid bottleneck, against the saved
originals on the same inputs.

  * CPU: the new C-ABI symbols are declared and typed, install / uninstall restore all three
    names, no local memory in the new kernels;
  * GPU: voxel grouping bit-identical to torch.unique(dim=0, return_inverse=True); the merge's features, coordinates
    and input gradient bit-identical to the dense original (M = 1, 2, 3; disjoint and overlapping subnets; all-zero,
    all-(−0.0) and NaN rows; negative coordinates) with its host synchronisations counted; the bottleneck against
    cuDNN fp32 (TF32 off) in train and eval mode with a negative global_min, output and every convolution and
    BatchNorm gradient; every fallback (spied); repeats and synchronisation counts; the KITTI-360 Net's 8-channel
    voxeliser; the unmodified Net's training and test steps with the other four hook groups on, trunk off and on.
GPU tests skip when oracle/_ref is not staged.
"""
import collections
import os
import re
import subprocess
import sys
import types
import warnings

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_eval as GE  # noqa: E402
import parity  # noqa: E402

STAGED = os.path.isdir(os.path.join(parity.REF, "pasco"))
needs_ref = pytest.mark.skipif(not STAGED, reason="oracle/_ref not staged")
K = 20
NEW_SYMBOLS = ("pasco_voxel_group", "pasco_voxel_group_order", "pasco_mimo_merge_cells", "pasco_mimo_merge_forward",
               "pasco_mimo_merge_backward")
KERNELS = ("k_vox_insert", "k_merge_insert", "k_collect", "k_rank", "k_vox_inverse", "k_merge_rows", "k_merge_copy",
           "k_merge_grad")


# ------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------
def test_new_symbols_declared_and_typed():
    from pasco_b200 import _lib
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "pasco_sm100.h")).read(), flags=re.S)
    for name in NEW_SYMBOLS:
        m = re.search(r"\b" + name + r"\s*\(([^;)]*)\)\s*;", src)
        assert m, f"{name} not declared"
        n_args = len([a for a in m.group(1).split(",") if a.strip()])
        assert name in _lib.PROTOTYPES and len(_lib.PROTOTYPES[name][1]) == n_args, name


def test_new_kernels_use_no_local_memory():
    from pasco_b200 import _lib, build
    build.build()
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    found = collections.Counter()
    for f in re.split(r"\n\s*Function : ", sass):
        head = f.split("\n")[0]
        if "voxel_cu" not in head:
            continue
        for n in KERNELS:
            if re.search(r"\d" + n + r"(E|I)", head):
                found[n] += 1
                assert not re.search(r"\b(LDL|STL)\b", f), f"{head}: local-memory traffic"
    assert set(found) == set(KERNELS), set(KERNELS) - set(found)


def _reference_modules():
    parity.reference_net()
    import importlib
    return (importlib.import_module("pasco.models.unet3d_sparse_v2"), importlib.import_module("pasco.models.augmenter"))


@needs_ref
def test_install_uninstall_restores_the_three_names():
    from pasco_b200 import hooks
    u, aug = _reference_modules()
    names = lambda: (u.CylinderFeat.forward, aug.Augmenter.merge, u.UNet3DV2.dense_bottleneck)  # noqa: E731
    before = names()
    assert hooks.install(attention=False, criterion=True)
    assert names() == before                                            # not requested: untouched
    for _ in range(2):
        assert hooks.install(attention=False, trunk=True)
    assert names() == (hooks._cylinder_forward, hooks._augmenter_merge, hooks._dense_bottleneck)
    assert u.CylinderFeat._pasco_b200_orig_forward is before[0]
    assert aug.Augmenter._pasco_b200_orig_merge is before[1]
    assert u.UNet3DV2._pasco_b200_orig_dense_bottleneck is before[2]
    for _ in range(2):
        hooks.uninstall()
    assert names() == before


# ------------------------------------------------------------------------------------------------
# GPU: voxel grouping
# ------------------------------------------------------------------------------------------------
def _rows(case, dtype, g):
    if case == "random_negative":
        r = torch.randint(-40, 40, (30_000, 4), generator=g)
        r[:, 0] = torch.randint(0, 3, (30_000,), generator=g)
        r = torch.cat([r, r[:5000]])                                   # duplicates
    elif case == "single_point":
        r = torch.tensor([[0, -7, 3, 32767]])
    elif case == "one_voxel":
        r = torch.tensor([[2, 5, -6, 7]]).repeat(1000, 1)
    elif case == "batches_0_7":
        r = torch.cat([torch.cat([torch.full((4000, 1), b), torch.randint(0, 30, (4000, 3), generator=g)], 1)
                       for b in range(8)])
    else:                                                              # P = 400 k, the reference's scene size
        r = torch.cat([torch.zeros(400_000, 1, dtype=torch.long), torch.randint(0, 256, (400_000, 2), generator=g),
                       torch.randint(-16, 32, (400_000, 1), generator=g)], 1)
    return r[torch.randperm(r.shape[0], generator=g)].to(dtype).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.int32, torch.int64])
@pytest.mark.parametrize("case", ["random_negative", "single_point", "one_voxel", "batches_0_7", "p400k"])
def test_voxel_group_matches_torch_unique(case, dtype):
    from pasco_b200 import ops
    rows = _rows(case, dtype, torch.Generator().manual_seed(3))
    want_u, want_i = torch.unique(rows, return_inverse=True, dim=0)
    got_u, got_i = ops.voxel_group(rows)
    assert got_u.dtype == want_u.dtype and got_i.dtype == want_i.dtype == torch.int64
    assert torch.equal(got_u, want_u) and torch.equal(got_i, want_i)


@pytest.mark.gpu
def test_voxel_group_flags_unpackable_rows():
    from pasco_b200 import ops
    rows = torch.tensor([[0, 1, 2, 3], [0, 40000, 0, 0]], device="cuda")
    assert ops.voxel_group(rows) is None
    assert ops.voxel_group(rows.int() * torch.tensor([1, 0, 1, 1], dtype=torch.int32, device="cuda")) is not None


# ------------------------------------------------------------------------------------------------
# GPU: the merge
# ------------------------------------------------------------------------------------------------
@pytest.fixture
def ref():
    from pasco_b200 import hooks
    u, aug = _reference_modules()
    import MinkowskiEngine as ME
    from pasco.models.layers import SPCDense3Dv2
    hooks.uninstall()
    assert hooks.install(attention=False, trunk=True)
    try:
        yield dict(ME=ME, u=u, aug=aug, SPCDense3Dv2=SPCDense3Dv2)
    finally:
        hooks.uninstall()


def _merge_input(M, overlap, seed, f=64, lo=-20):
    g = torch.Generator().manual_seed(seed)
    per = []
    for t in range(M):
        cells = torch.unique(torch.randint(lo, lo + 30, (3000, 3), generator=g), dim=0)
        if not overlap:
            cells[:, 0] += 40 * t
        per.append(torch.cat([torch.full((cells.shape[0], 1), t), cells], 1))
    C = torch.cat(per).int()
    F = torch.randn(C.shape[0], f, generator=g)
    F[::7] = 0.0                               # rows that are zero in their subnet (and often in every subnet)
    F[3::11] = -0.0
    F[5, 3] = float("nan")
    return F.cuda(), C.cuda()


def _merge_both(r, F, C):
    """(features, coordinates, input gradient) of the original and of the hook."""
    ME = r["ME"]
    aug = r["aug"].Augmenter()
    out = []
    for fn in (r["aug"].Augmenter._pasco_b200_orig_merge, r["aug"].Augmenter.merge):
        x = F.clone().requires_grad_(True)
        y = fn(aug, ME.SparseTensor(x, C))
        w = torch.randn(y.F.shape, generator=torch.Generator().manual_seed(1)).cuda()
        (y.F * w).nan_to_num().sum().backward()
        out.append((y.F.detach(), y.C, x.grad))
    return out


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("M", [1, 2, 3])
@pytest.mark.parametrize("overlap", [False, True])
def test_merge_bit_identical_to_the_original(ref, M, overlap):
    F, C = _merge_input(M, overlap, seed=M + 10 * overlap)
    (fa, ca, ga), (fb, cb, gb) = _merge_both(ref, F, C)
    for name, a_, b_ in (("features", fa, fb), ("gradient", ga, gb)):
        if a_.shape == b_.shape and not torch.equal(a_.view(torch.int32), b_.view(torch.int32)):
            at = torch.nonzero(a_.view(torch.int32) != b_.view(torch.int32))
            print(name, "differs at", at[:4].tolist(), "of", at.shape[0], a_[tuple(at[0])].item(), b_[tuple(at[0])].item())
    assert torch.equal(ca.int(), cb.int())
    assert fa.shape == fb.shape and torch.equal(fa.view(torch.int32), fb.view(torch.int32))     # NaN and −0.0 bits too
    assert torch.equal(ga.view(torch.int32), gb.view(torch.int32))
    assert (ca[:, 1:] < 0).any()                                        # negative min_coordinate


def _syncs(fn):
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            out = fn()
        finally:
            torch.cuda.set_sync_debug_mode("default")
    return out, [f"{os.path.basename(v.filename)}:{v.lineno}" for v in w if "called a synchronizing" in str(v.message)]


@pytest.mark.gpu
@needs_ref
def test_merge_reads_only_its_row_count_on_the_host(ref):
    """No synchronisation for the minimum coordinate: the one crossing reads the merged row count, the subnet count
    and the range flag together, whatever M and N."""
    ME = ref["ME"]
    aug = ref["aug"].Augmenter()
    counts = {}
    for M, seed in ((2, 1), (3, 2)):
        F, C = _merge_input(M, True, seed)
        x = ME.SparseTensor(F, C)
        _, sites = _syncs(lambda: aug.merge(x))
        counts[M] = sites
    assert all(len(s) == 1 for s in counts.values()), counts
    assert len({tuple(s) for s in counts.values()}) == 1, counts


# ------------------------------------------------------------------------------------------------
# GPU: the dense bottleneck
# ------------------------------------------------------------------------------------------------
def _bottleneck_input(r, gmin, seed, c=256, size=(32, 32, 4), scale=8):
    g = torch.Generator().manual_seed(seed)
    occ = torch.rand(size, generator=g) < 0.3
    cells = torch.nonzero(occ)
    C = torch.cat([torch.zeros(cells.shape[0], 1, dtype=torch.long), cells * scale + torch.tensor(gmin)], 1).int()
    F = torch.randn(cells.shape[0], c, generator=g)
    gmax = torch.tensor(gmin) + torch.tensor(size) * scale - 1
    return F.cuda(), C.cuda(), torch.tensor(gmin).cuda(), gmax.cuda()


def _unet(r, train, seed=0):
    torch.manual_seed(seed)
    U = r["u"].UNet3DV2
    u = U.__new__(U)                                  # only dense3d: what dense_bottleneck reads
    torch.nn.Module.__init__(u)
    u.dense3d = torch.nn.Sequential(r["SPCDense3Dv2"](init_size=256), torch.nn.Dropout3d(0.0)).cuda()
    for m in u.dense3d.modules():
        if isinstance(m, torch.nn.BatchNorm3d):
            m.weight.data.uniform_(0.5, 1.5)
            m.bias.data.uniform_(-0.2, 0.2)
            m.running_mean.uniform_(-0.1, 0.1)
            m.running_var.uniform_(0.5, 2.0)
    u.train(train)
    return u


def _bottleneck_run(r, u, fn, F, C, gmin, gmax, scale=8):
    ME = r["ME"]
    for p in u.parameters():
        p.grad = None
    x = F.clone().requires_grad_(True)
    cm = ME.CoordinateManager()
    deep = ME.SparseTensor(x, C, tensor_stride=scale, coordinate_manager=cm)
    y = fn(u, deep, 1, gmin, gmax)
    w = torch.randn(y.F.shape, generator=torch.Generator().manual_seed(2)).cuda()
    (y.F * w).sum().backward()
    grads = {n: p.grad.detach().clone() for n, p in u.named_parameters()}
    return y.F.detach(), y.C, grads, x.grad, y.coordinate_manager is cm


def _maxabs(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max().clamp(min=1e-30))


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("train", [True, False])
@pytest.mark.parametrize("gmin", [(0, 0, 0), (-24, 16, -8)])
def test_bottleneck_matches_cudnn(ref, train, gmin):
    from pasco_b200 import ops
    ops.set_precision("fp32")                         # cuDNN fp32, TF32 off
    F, C, gmn, gmx = _bottleneck_input(ref, gmin, seed=4)
    U = ref["u"].UNet3DV2
    want = _bottleneck_run(ref, _unet(ref, train), U._pasco_b200_orig_dense_bottleneck, F, C, gmn, gmx)
    got = _bottleneck_run(ref, _unet(ref, train), U.dense_bottleneck, F, C, gmn, gmx)
    assert got[4] and want[4]
    assert torch.equal(got[1].int(), want[1].int())
    assert set(got[2]) == set(want[2]) and sum("conv" in n or "res_" in n for n in got[2]) >= 11
    grads = {"x": (got[3], want[3]), **{n: (got[2][n], want[2][n]) for n in want[2]}}
    maxabs = {n: _maxabs(a_, b_) for n, (a_, b_) in grads.items()}
    rel = {n: float((a_ - b_).double().norm() / b_.double().norm()) for n, (a_, b_) in grads.items()}
    worst = lambda d: {k: f"{v:.1e}" for k, v in sorted(d.items(), key=lambda kv: -kv[1])[:4]}  # noqa: E731
    print(f"output max-abs normalised {_maxabs(got[0], want[0]):.1e}; gradients max-abs normalised {worst(maxabs)}, "
          f"relative L2 {worst(rel)}")
    # the output within 1e-3 of max |y|; the gradients within 1e-2 in relative L2 (ReLU and split-K rounding decide a
    # few rows differently, which moves single weight-gradient entries by more)
    assert _maxabs(got[0], want[0]) < 1e-3
    assert max(rel.values()) < 1e-2, rel


# ------------------------------------------------------------------------------------------------
# GPU: fallbacks
# ------------------------------------------------------------------------------------------------
def _spy(cls, attr, calls):
    orig = getattr(cls, attr)
    setattr(cls, attr, lambda *a, **k: calls.append(attr) or "orig")
    return orig


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("case", ["fea_compre", "cpu", "out_of_range"])
def test_cylinder_fallbacks(ref, case):
    u = ref["u"]
    torch.manual_seed(0)
    cf = u.CylinderFeat(fea_dim=8, out_pt_fea_dim=16, fea_compre=4 if case == "fea_compre" else None)
    dev = "cpu" if case == "cpu" else "cuda"
    cf.to(dev)
    ind = torch.randint(0, 20, (100, 3), device=dev)
    if case == "out_of_range":
        ind[7, 1] = 70000
    calls = []
    orig = _spy(u.CylinderFeat, "_pasco_b200_orig_forward", calls)
    try:
        out = cf([torch.randn(100, 8, device=dev)], [ind])
    finally:
        u.CylinderFeat._pasco_b200_orig_forward = orig
    assert calls == ["_pasco_b200_orig_forward"] and out == "orig"


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("case", ["cpu", "nine_subnets"])
def test_merge_fallbacks(ref, case):
    ME, aug = ref["ME"], ref["aug"]
    F, C = _merge_input(9 if case == "nine_subnets" else 2, True, 0)
    x = types.SimpleNamespace(F=F.cpu(), C=C.cpu()) if case == "cpu" else ME.SparseTensor(F, C)
    calls = []
    orig = _spy(aug.Augmenter, "_pasco_b200_orig_merge", calls)
    try:
        out = aug.Augmenter().merge(x)
    finally:
        aug.Augmenter._pasco_b200_orig_merge = orig
    assert calls == ["_pasco_b200_orig_merge"] and out == "orig"


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("case", ["bs2", "no_dropout", "dropout_train", "cpu"])
def test_bottleneck_fallbacks(ref, case):
    ME, U = ref["ME"], ref["u"].UNet3DV2
    F, C, gmn, gmx = _bottleneck_input(ref, (0, 0, 0), seed=1)
    u = _unet(ref, True)
    if case == "no_dropout":
        u.dense3d = torch.nn.Sequential(u.dense3d[0])
    if case == "dropout_train":
        u.dense3d[1].p = 0.2
    if case == "cpu":
        F, C, gmn, gmx = F.cpu(), C.cpu(), gmn.cpu(), gmx.cpu()
    deep = (types.SimpleNamespace(F=F, C=C, tensor_stride=[8, 8, 8]) if case == "cpu"
            else ME.SparseTensor(F, C, tensor_stride=8))
    calls = []
    orig = _spy(U, "_pasco_b200_orig_dense_bottleneck", calls)
    try:
        out = U.dense_bottleneck(u, deep, 2 if case == "bs2" else 1, gmn, gmx)
        if case == "dropout_train":                  # eval mode: the Dropout3d is the identity, the hook runs
            u.eval()
            out2 = U.dense_bottleneck(u, deep, 1, gmn, gmx)
            assert out2 != "orig"
    finally:
        U._pasco_b200_orig_dense_bottleneck = orig
    assert calls == ["_pasco_b200_orig_dense_bottleneck"] and out == "orig"


# ------------------------------------------------------------------------------------------------
# GPU: repeats and host synchronisations
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@needs_ref
def test_repeats_bit_identical_and_syncs_constant(ref):
    from pasco_b200 import hooks, ops
    ops.set_precision("fp32")
    ME, u = ref["ME"], ref["u"]
    counts = collections.defaultdict(set)
    for n_pts, M in ((20_000, 2), (200_000, 3)):
        torch.manual_seed(0)
        cf = u.CylinderFeat(fea_dim=283, out_pt_fea_dim=64).cuda().eval()
        g = torch.Generator().manual_seed(n_pts)
        fea = [torch.randn(n_pts, 283, generator=g).cuda() for _ in range(M)]
        ind = [torch.randint(0, 128, (n_pts, 3), generator=g).cuda() for _ in range(M)]
        F, C = _merge_input(M, True, n_pts)
        Fb, Cb, gmn, gmx = _bottleneck_input(ref, (-8, 0, 8), seed=n_pts)
        unet = _unet(ref, False)
        x, deep = ME.SparseTensor(F, C), ME.SparseTensor(Fb, Cb, tensor_stride=8)
        u.UNet3DV2.dense_bottleneck(unet, deep, 1, gmn, gmx)       # the grid's kernel maps are built once per size
        outs = []
        for _ in range(2):
            (cu, cp), s1 = _syncs(lambda: cf(fea, ind))
            m, s2 = _syncs(lambda: ref["aug"].Augmenter().merge(x))
            b, s3 = _syncs(lambda: u.UNet3DV2.dense_bottleneck(unet, deep, 1, gmn, gmx))
            counts["cylinder"].add(len(s1))
            counts["merge"].add(len(s2))
            counts["bottleneck"].add(len(s3))
            outs.append((cu, cp, m.F, m.C, b.F, b.C))
        for a_, b_ in zip(*outs):                   # bit for bit (the merge input holds a NaN)
            assert a_.shape == b_.shape and a_.contiguous().view(torch.uint8).equal(b_.contiguous().view(torch.uint8))
    print("host synchronisations per hooked call:", dict(counts))
    for k, v in counts.items():
        assert len(v) == 1 and max(v) <= hooks.TRUNK_SYNCS, (k, v)


# ------------------------------------------------------------------------------------------------
# GPU: the KITTI-360 Net's voxeliser (8-channel point features) and merge
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@needs_ref
def test_kitti360_voxeliser_and_merge(ref):
    from pasco.models.net_panoptic_sparse_kitti360 import Net_kitti360
    from pasco_b200.synthetic import make_scene
    ME = ref["ME"]
    torch.manual_seed(0)
    net = Net_kitti360(n_classes=19, class_names=[str(i) for i in range(19)], class_weights=torch.ones(19),
                       encoder_dropouts=[0.0] * 3, decoder_dropouts=[0.0] * 3, dense3d_dropout=0.0, n_infers=3,
                       class_frequencies={f"1_{s}": np.ones(19) for s in (1, 2, 4)}, in_channels=8, f=64).cuda().eval()
    sc = make_scene((64, 64, 8), 0.08, 3, in_ch=8, n_classes=19, seed=16)
    fea, ind = [t.cuda() for t in sc["in_feats"]], [t.cuda() for t in sc["in_coords"]]
    outs = []
    for fn in (type(net.feat)._pasco_b200_orig_forward, type(net.feat).forward):
        torch.manual_seed(0)
        c, f = fn(net.feat, fea, ind)
        merged = net.augmenter.merge(ME.SparseTensor(f, c.int()))
        outs.append((c, f, merged.F, merged.C, torch.rand(1, device="cuda")))
    (c0, f0, m0, mc0, r0), (c1, f1, m1, mc1, r1) = outs
    assert torch.equal(c0, c1) and torch.equal(mc0, mc1)
    assert torch.equal(r0, r1), "the CUDA generator moved differently"
    # eval mode: the point order reaches no statistics; the MLP's rows may round differently in another order
    assert torch.allclose(f0, f1, rtol=1e-5, atol=1e-6) and torch.allclose(m0, m1, rtol=1e-5, atol=1e-6)


# ------------------------------------------------------------------------------------------------
# GPU: the unmodified Net end to end, the other four hook groups on
# ------------------------------------------------------------------------------------------------
class _Coords:
    """The coordinate sets the transformer receives at every decoder scale, per call."""

    def __init__(self):
        from pasco.models.transformer.transformer_predictor_v2 import TransformerPredictorV2
        self.cls, self.got = TransformerPredictorV2, []

    def __enter__(self):
        inner = self.cls.forward

        def rec(this, xs, *a, **k):
            self.got.append({s: np.unique(xs[s][1].reshape(-1, 4).cpu().numpy(), axis=0) for s in xs})
            return inner(this, xs, *a, **k)
        self.inner = inner
        self.cls.forward = rec
        return self

    def __exit__(self, *exc):
        self.cls.forward = self.inner


def _set(hooks, trunk):
    hooks.uninstall()
    assert hooks.install(attention=True, postprocess=True, evaluate=True, criterion=True, trunk=trunk)


def _same_coords(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert set(x) == set(y)
        for s in x:
            assert np.array_equal(x[s], y[s]), f"scale {s}"


def _val(v):
    return float(v.detach()) if torch.is_tensor(v) else float(v)


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("M", [1, 2])
def test_net_training_step_trunk_off_and_on(ref, M):
    from pasco_b200 import hooks, ops
    from recipe import fill_state_dict
    ops.set_precision("fp32")
    hooks.uninstall()
    _, net = parity.reference_net(n_infers=M)
    net.class_weights = [torch.ones(K + 1) for _ in range(M)]
    net.criterion.class_weights = net.class_weights
    net.criterion.compl_labelweights = torch.ones(K)
    net.load_state_dict(fill_state_dict(net.state_dict()))
    net.object_mask_threshold = 0.05
    dev = torch.device("cuda")
    net.to(dev).train()
    meta = parity.INFER_MANIFEST["cases"]["m2" if M == 2 else "m1"]
    sc = parity.scene(meta, M)
    grid = tuple(meta["grid"])
    g = torch.Generator().manual_seed(5)
    sem = torch.randint(0, K, (M,) + grid, generator=g)
    sem[torch.rand(sem.shape, generator=g) < 0.6] = 0
    sem[:, :, :2, :] = 255
    mask_label = []
    for m in range(M):
        present = [c for c in range(1, K) if (sem[m] == c).any()]
        mask_label.append({"labels": torch.tensor(present, dtype=torch.uint8, device=dev),
                           "masks": torch.stack([sem[m] == c for c in present]).to(dev)})
    batch = dict(in_feats=sc["in_feats"], in_coords=sc["in_coords"], min_Cs=[t.to(dev) for t in sc["min_Cs"]],
                 max_Cs=[t.to(dev) for t in sc["max_Cs"]], Ts=[t.to(dev) for t in sc["Ts"]],
                 global_min_Cs=sc["global_min_Cs"].to(dev), global_max_Cs=sc["global_max_Cs"].to(dev),
                 sem_labels=sc["sem_labels"], semantic_label=sem.to(torch.uint8).to(dev),
                 geo_labels={"1_1": torch.where(sem == 255, 255.0, (sem > 0).float()).to(dev)}, mask_label=mask_label)

    def step(trunk):
        _set(hooks, trunk)
        logged = {}
        net.log = lambda k, v, **kw: logged.__setitem__(k, _val(v))
        net.zero_grad(set_to_none=True)
        torch.manual_seed(0)
        with _Coords() as rec:
            out = net.step(batch, "train")
        out["loss"].backward()
        return _val(out["loss"]), logged, rec.got

    try:
        want = step(False)
        got = step(True)
    finally:
        hooks.uninstall()
    _same_coords(got[2], want[2])
    assert set(got[1]) == set(want[1])
    for k, v in want[1].items():
        assert abs(got[1][k] - v) <= 1e-3 * max(1.0, abs(v)), (k, got[1][k], v)
    print(f"M = {M}: loss {got[0]:.6f} (trunk on) vs {want[0]:.6f} (off)")


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("M", [1, 3])
def test_net_step_inference_trunk_off_and_on(ref, M, capsys):
    from pasco_b200 import hooks, ops
    from recipe import fill_state_dict
    ops.set_precision("fp32")
    hooks.uninstall()
    _, net = parity.reference_net(n_infers=M)
    if M == 1:
        net, _ = parity.load_eval(net, "m1", ref_names=False)
    else:
        net.load_state_dict(fill_state_dict(net.state_dict()))
        net.cuda().eval()
    net.object_mask_threshold = 0.05
    dev = torch.device("cuda")
    sc = parity.scene(parity.INFER_MANIFEST["cases"]["m1"], M)
    sem, ml = GE.gt_scene(0)
    ml = {"labels": ml["labels"].to(dev), "masks": ml["masks"].to(dev)}
    batch = dict(in_feats=sc["in_feats"], in_coords=sc["in_coords"], min_Cs=[t.to(dev) for t in sc["min_Cs"]],
                 max_Cs=[t.to(dev) for t in sc["max_Cs"]], Ts=[t.to(dev) for t in sc["Ts"]],
                 global_min_Cs=sc["global_min_Cs"].to(dev), global_max_Cs=sc["global_max_Cs"].to(dev),
                 geo_labels=sc["sem_labels"], mask_classes=sc["mask_classes"],
                 semantic_label=sem.unsqueeze(0).to(dev), semantic_label_origin=sem.unsqueeze(0).to(dev),
                 mask_label=[ml], mask_label_origin=[ml])
    from pasco.loss.panoptic_quality import PQStat
    from pasco.models.metrics import SSCMetrics, UncertaintyMetrics

    def run(trunk):
        _set(hooks, trunk)
        for i in net.pq_stat["test"]:
            net.pq_stat["test"][i] = PQStat()
            net.ssc_metrics["test"][i] = SSCMetrics(net.n_classes)
            net.uncertainty_metrics["test"][i] = UncertaintyMetrics()
            net.uncertainty_metrics_by_thresholds[0.5][i] = UncertaintyMetrics()
        torch.manual_seed(0)
        with _Coords() as rec, torch.no_grad():
            net.step_inference(batch, "test", eval=True)
        ssc = {i: (m.completion_tp, m.completion_fp, m.completion_fn, m.tps.tolist())
               for i, m in net.ssc_metrics["test"].items()}
        pq = {i: {c: (s.tp, s.fp, s.fn) for c, s in p.pq_per_cat.items()} for i, p in net.pq_stat["test"].items()}
        return rec.got, ssc, pq

    try:
        want = run(False)
        got = run(True)
    finally:
        hooks.uninstall()
    _same_coords(got[0], want[0])
    assert got[1] == want[1]
    assert got[2] == want[2]
