"""The criterion hook (pasco_b200/hooks.py install(criterion=True)): the unmodified reference's
SetCriterion.compute_losses and completion losses on csrc/setloss.cu, against the stored outputs of the reference's own
loss code (tests/golden/loss_m2.npz) and against the saved originals on the same inputs.

  * CPU: the new C-ABI symbols are declared and typed, install / uninstall restore all three
    replaced names, no local memory in the new kernels;
  * GPU: the fixture (M = 2, 4 levels, overlapping masks, unknown rows, 255 labels, dustbin queries); N = 400 k rows,
    Q = 100, T = 30 against the original (cost matrices, assignments, every term, gradients), and with two target words
    (T = 40) and 40 classes (class 31 present, 32..39 absent); Lovász with ties, an empty present set and all rows left
    out; T = 0, no valid row, no kept query; every fallback of the criterion and of the completion loss (spied);
    bit-identical repeats and every host synchronisation counted, independent of N, with the class weights on the host
    as the reference keeps them; the unmodified Net's training step with and without the hook.
GPU tests skip when oracle/_ref is not staged.
"""
import collections
import os
import re
import subprocess
import sys
import warnings

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import parity  # noqa: E402

STAGED = os.path.isdir(os.path.join(parity.REF, "pasco"))
needs_ref = pytest.mark.skipif(not STAGED, reason="oracle/_ref not staged")
GOLD = os.path.join(HERE, "golden", "loss_m2.npz")
M, LEVELS, K = 2, 4, 20
WEIGHTS = {"ssc_ce": 0.3, "ssc_lovasz": 1.0, "loss_ce": 2.0, "loss_mask": 20.0, "loss_dice": 1.0}
NEW_SYMBOLS = ("pasco_setloss_sample", "pasco_setloss_match_cost", "pasco_setloss_pair_sums",
               "pasco_setloss_pair_backward", "pasco_setloss_ssc_forward", "pasco_setloss_ssc_backward",
               "pasco_lovasz_errors", "pasco_lovasz_grad", "pasco_lovasz_backward")
TERMS = ("loss_ce", "loss_mask", "loss_dice", "ssc_ce_loss", "ssc_lovasz_loss")


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
    names = ("k_sl_sample", "k_sl_reduce", "k_sl_cost", "k_sl_cost_finish", "k_sl_pair_sums", "k_sl_pair_backward",
             "k_sl_ssc_forward", "k_sl_ssc_backward", "k_lov_errors", "k_lov_tile_counts", "k_lov_tile_scan",
             "k_lov_grad", "k_lov_class_sum", "k_lov_scatter", "k_lov_softmax_backward")
    found = collections.Counter()
    for f in re.split(r"\n\s*Function : ", sass):
        head = f.split("\n")[0]
        for n in names:
            if re.search(r"\d" + n + r"E", head):
                found[n] += 1
                assert not re.search(r"\b(LDL|STL)\b", f), f"{head}: local-memory traffic"
    assert set(found) == set(names), set(names) - set(found)


def _reference_modules():
    parity.reference_net()
    import importlib
    return (importlib.import_module("pasco.models.net_panoptic_sparse"),
            importlib.import_module("pasco.models.net_panoptic_sparse_kitti360"),
            importlib.import_module("pasco.loss.criterion_sparse"))


@needs_ref
def test_install_uninstall_restores_the_three_names():
    from pasco_b200 import hooks
    nps, k360, cs = _reference_modules()
    before = (cs.SetCriterion.compute_losses, nps.compute_sem_compl_loss, k360.compute_sem_compl_loss_kitti360)
    assert hooks.install(attention=False)
    assert cs.SetCriterion.compute_losses is before[0]                 # not requested: untouched
    for _ in range(2):
        assert hooks.install(attention=False, criterion=True)
    assert cs.SetCriterion.compute_losses is hooks._compute_losses
    assert nps.compute_sem_compl_loss is hooks._compute_sem_compl_loss
    assert k360.compute_sem_compl_loss_kitti360 is hooks._compute_sem_compl_loss_kitti360
    assert nps._pasco_b200_orig_compute_sem_compl_loss is before[1]
    for _ in range(2):
        hooks.uninstall()
    assert (cs.SetCriterion.compute_losses, nps.compute_sem_compl_loss, k360.compute_sem_compl_loss_kitti360) == before


# ------------------------------------------------------------------------------------------------
# GPU helpers
# ------------------------------------------------------------------------------------------------
@pytest.fixture
def ref():
    from pasco_b200 import hooks
    nps, k360, cs = _reference_modules()
    from pasco.loss import losses, matcher_sparse
    import MinkowskiEngine as ME
    assert hooks.install(attention=False, criterion=True)
    try:
        yield dict(ME=ME, nps=nps, k360=k360, cs=cs, losses=losses, matcher=matcher_sparse)
    finally:
        hooks.uninstall()


def _criterion(r, class_weights, compl_labelweights, dev="cuda"):
    """The reference's SetCriterion; the per-subnet class weights stay on the host, where the reference keeps them."""
    matcher = r["matcher"].HungarianMatcher(cost_class=1.0, cost_mask=WEIGHTS["loss_mask"],
                                            cost_dice=WEIGHTS["loss_dice"])
    return r["cs"].SetCriterion(len(compl_labelweights), matcher=matcher, weight_dict=dict(WEIGHTS), eos_coef=0.1,
                                class_weights=[w.cpu() for w in class_weights],
                                compl_labelweights=compl_labelweights.to(dev)).to(dev)


class _Assignments:
    """Records every linear_sum_assignment result: the original's (matcher module's name) and the hook's (scipy's)."""

    def __init__(self, r, monkeypatch):
        import scipy.optimize
        self.got = []
        real = scipy.optimize.linear_sum_assignment

        def rec(c):
            out = real(c)
            self.got.append((np.asarray(c, dtype=np.float32).copy(), out))
            return out
        monkeypatch.setattr(scipy.optimize, "linear_sum_assignment", rec)
        monkeypatch.setattr(r["matcher"], "linear_sum_assignment", rec)


def _run(r, crit, pred, target, sem, unknown, i_infer, min_C, hooked):
    """SetCriterion.forward with the hook or the saved original, the spy counting the hook's fallbacks."""
    cls = r["cs"].SetCriterion
    falls = []
    orig = cls._pasco_b200_orig_compute_losses
    if hooked:
        cls._pasco_b200_orig_compute_losses = lambda *a, **k: falls.append(1) or orig(*a, **k)
    else:
        cls.compute_losses = orig
    try:
        out = crit(None, pred, target, sem, unknown, i_infer, [], min_C)
    finally:
        cls._pasco_b200_orig_compute_losses = orig
        cls.compute_losses = __import__("pasco_b200.hooks", fromlist=["x"])._compute_losses
    return out, falls


def _flat(ls):
    out = {k: ls[k] for k in TERMS}
    out.update(ls["loss_aux"])
    return out


def _val(v):
    return float(v) if not torch.is_tensor(v) else float(v.detach())


# ------------------------------------------------------------------------------------------------
# GPU: the fixture
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@needs_ref
def test_fixture_terms_and_assignments(ref, monkeypatch):
    g = dict(np.load(GOLD))
    ME, dev = ref["ME"], torch.device("cuda")
    crit = _criterion(ref, list(torch.as_tensor(g["class_weights"])), torch.as_tensor(g["compl_labelweights"]))
    rec = _Assignments(ref, monkeypatch)
    sem_all = torch.as_tensor(g["semantic_label"]).to(dev)
    for m in range(M):
        def level(lv):
            return {"voxel_logits": ME.SparseTensor(torch.as_tensor(g[f"vox_F_m{m}_l{lv}"]).to(dev),
                                                    torch.as_tensor(g[f"vox_C_m{m}"]).to(dev)),
                    "query_logits": torch.as_tensor(g[f"query_m{m}_l{lv}"]).to(dev)}
        pred = level(0)
        pred["aux_outputs"] = [level(lv) for lv in range(1, LEVELS)]
        target = [{"labels": torch.as_tensor(g["labels"][m]).to(dev), "masks": torch.as_tensor(g["masks"][m]).to(dev)}]
        sem = sem_all[m].unsqueeze(0)
        rec.got.clear()
        ls, falls = _run(ref, crit, pred, target, sem, sem == 255, m, torch.as_tensor(g["min_C"]).to(dev), True)
        assert falls == [], "the hook fell back"
        assert len(rec.got) == LEVELS
        for lv, (_, (qi, tj)) in enumerate(rec.got):
            assert np.array_equal(np.stack([qi, tj]), g[f"match_m{m}_l{lv}"]), f"assignment m{m} level {lv}"
        flat = _flat(ls)
        assert len(flat) == len(TERMS) + 5 * (LEVELS - 1)
        for k, v in flat.items():
            want = float(g[f"{k}_m{m}"])
            assert abs(_val(v) - want) <= 1e-4 * max(1.0, abs(want)), (k, m, _val(v), want)

    sem_at = {s: [ME.SparseTensor(torch.as_tensor(g[f"sem{s}_F_m{m}"]).to(dev), torch.as_tensor(g[f"sem{s}_C_m{m}"]).to(dev))
                  for m in range(M)] for s in (1, 2, 4)}
    labels = {f"1_{s}": torch.as_tensor(g[f"sem_labels_1_{s}"]).to(dev) for s in (1, 2, 4)}
    freqs = {f"1_{s}": g["class_frequencies"][i] for i, s in enumerate((1, 2, 4))}
    mins, maxs = [torch.as_tensor(g["min_C"]).to(dev)] * M, [torch.as_tensor(g["max_C"]).to(dev)] * M
    from pasco_b200 import hooks
    for fn, sfx in ((hooks._compute_sem_compl_loss, ""), (hooks._compute_sem_compl_loss_kitti360, "_kitti360")):
        calls = []
        saved = hooks._orig_compl[:]
        hooks._orig_compl[:] = [lambda *a: calls.append(1) or saved[0](*a), lambda *a: calls.append(1) or saved[1](*a)]
        try:
            ce, lov = fn(labels, sem_at, mins, maxs, freqs)
        finally:
            hooks._orig_compl[:] = saved
        assert calls == []
        for got, k in ((ce, "compl_ce"), (lov, "compl_lovasz")):
            want = float(g[k + sfx])
            assert abs(float(got) - want) <= 1e-4 * max(1.0, abs(want)), (k + sfx, float(got), want)


# ------------------------------------------------------------------------------------------------
# GPU: at scale, against the original on the same inputs
# ------------------------------------------------------------------------------------------------
def _scale_inputs(r, N=400_000, Q=100, T=30, seed=0, dev="cuda", K=K, sem_classes=None):
    """N rows of a 256 x 256 x 32 volume, T overlapping boxes, unknown slab, 255 labels, a few dustbin queries; K
    classes, semantic labels in [0, sem_classes or K)."""
    g = torch.Generator().manual_seed(seed)
    X, Y, Z = 256, 256, 32
    cells = torch.randperm(X * Y * Z, generator=g)[:N]
    C = torch.stack([torch.zeros_like(cells), cells // (Y * Z), (cells // Z) % Y, cells % Z], 1).int()
    masks = torch.zeros(T, X, Y, Z, dtype=torch.bool)
    labels = torch.randint(1, K, (T,), generator=g).to(torch.uint8)
    for t in range(T):
        lo = [int(torch.randint(0, s - s // 4, (1,), generator=g)) for s in (X, Y, Z)]
        hi = [l + max(2, s // 4) for l, s in zip(lo, (X, Y, Z))]
        masks[t, lo[0]:hi[0], lo[1]:hi[1], lo[2]:hi[2]] = True
    sem = torch.randint(0, sem_classes or K, (1, X, Y, Z), generator=g).to(torch.uint8)
    sem[:, :, 240:, :] = 255
    F = torch.randn(N, Q, generator=g) * 3
    ql = torch.randn(1, Q, K + 1, generator=g)
    ql[0, :10, K] += 8.0
    cw = torch.ones(K + 1)
    cw[1:K] = 0.5 + torch.rand(K - 1, generator=g)
    d = lambda t: t.to(dev)  # noqa: E731
    return dict(F=d(F), C=d(C), ql=d(ql), masks=d(masks), labels=d(labels), sem=d(sem), unknown=d(sem == 255),
                cw=cw, lw=0.5 + torch.rand(K, generator=g))


def _one_level(r, crit, x, hooked):
    F = x["F"].clone().requires_grad_(True)
    ql = x["ql"].clone().requires_grad_(True)
    pred = {"voxel_logits": r["ME"].SparseTensor(F, x["C"]), "query_logits": ql}
    target = [{"labels": x["labels"], "masks": x["masks"]}]
    ls, falls = _run(r, crit, pred, target, x["sem"], x["unknown"], 0, torch.zeros(3, dtype=torch.long, device="cuda"),
                     hooked)
    total = sum(v for k, v in ls.items() if k in TERMS and torch.is_tensor(v))
    total.backward()
    return {k: _val(ls[k]) for k in TERMS}, F.grad, ql.grad, falls


@pytest.mark.gpu
@needs_ref
def test_at_scale_against_the_original(ref, monkeypatch):
    x = _scale_inputs(ref)
    crit = _criterion(ref, [x["cw"]], x["lw"])
    rec = _Assignments(ref, monkeypatch)
    want = _one_level(ref, crit, x, False)
    (C_want, (qi_w, tj_w)), = rec.got
    rec.got.clear()
    got = _one_level(ref, crit, x, True)
    (C_got, (qi_g, tj_g)), = rec.got
    assert got[3] == [], "the hook fell back"
    scale = float(np.abs(C_want).max())
    assert float(np.abs(C_got - C_want).max()) <= 1e-5 * scale
    same = np.array_equal(qi_g, qi_w) and np.array_equal(tj_g, tj_w)
    if not same:          # a tie: both assignments cost the same under either matrix, within the tolerance
        for Cm in (C_want, C_got):
            assert abs(Cm[qi_g, tj_g].sum() - Cm[qi_w, tj_w].sum()) <= 1e-5 * scale * len(qi_w)
    for k in TERMS:
        assert abs(got[0][k] - want[0][k]) <= 1e-4 * max(1.0, abs(want[0][k])), (k, got[0][k], want[0][k])
    if same:
        for a, b in ((got[1], want[1]), (got[2], want[2])):
            assert float((a - b).norm() / b.norm()) <= 1e-3
    print("terms", got[0], "assignments equal:", same)


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("case", ["T30", "T40", "K40"])
def test_gradients_with_the_originals_indices(ref, monkeypatch, case):
    """The original's assignment injected into the hook (scipy returns it): every term and the gradients w.r.t.
    voxel_logits.F and query_logits agree.  T40: two target words per row.  K40: 40 classes, semantic labels in
    [0, 32) with class 31 present, so classes 32..39 are absent from the ssc Lovász term."""
    import scipy.optimize
    if case == "K40":
        x = _scale_inputs(ref, N=100_000, seed=1, K=40, sem_classes=32)
        x["sem"][:, :4] = 31
    else:
        x = _scale_inputs(ref, N=100_000, seed=1, T=40 if case == "T40" else 30)
    crit = _criterion(ref, [x["cw"]], x["lw"])
    rec = _Assignments(ref, monkeypatch)
    want = _one_level(ref, crit, x, False)
    fixed = rec.got[0][1]
    monkeypatch.setattr(scipy.optimize, "linear_sum_assignment", lambda c: fixed)
    got = _one_level(ref, crit, x, True)
    assert got[3] == []
    for k in TERMS:
        assert abs(got[0][k] - want[0][k]) <= 1e-4 * max(1.0, abs(want[0][k])), (case, k, got[0][k], want[0][k])
    for a, b, name in ((got[1], want[1], "voxel_logits.F"), (got[2], want[2], "query_logits")):
        err = float((a - b).norm() / b.norm())
        assert err <= 1e-3, (case, name, err)


# ------------------------------------------------------------------------------------------------
# GPU: edge cases
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@needs_ref
def test_lovasz_edge_cases(ref):
    from pasco_b200 import ops
    from pasco.loss.lovasz import lovasz_softmax_flat
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(3)
    # ties: logits on a coarse grid, many rows with identical errors
    x = (torch.randint(-2, 3, (5000, 6), generator=g).float()).to(dev).requires_grad_(True)
    lab = torch.randint(0, 6, (5000,), generator=g).to(dev)
    lab[:50] = 255
    want = lovasz_softmax_flat(x[lab != 255], lab[lab != 255], ignores=[0])
    lab_i = torch.where(lab == 255, -1, lab).to(torch.int32)
    present = torch.tensor([False] + [True] * 5, device=dev)
    got = ops.lovasz_softmax(x, lab_i, present)
    assert abs(float(got) - float(want)) <= 1e-5, (float(got), float(want))
    # no ties: gradients
    y = torch.randn(5000, 6, generator=g).to(dev).requires_grad_(True)
    want = lovasz_softmax_flat(y[lab != 255], lab[lab != 255], ignores=[0])
    gw, = torch.autograd.grad(want, y)
    got = ops.lovasz_softmax(y, lab_i, present)
    gg, = torch.autograd.grad(got, y)
    assert abs(float(got) - float(want)) <= 1e-5
    assert float((gg - gw).norm() / gw.norm()) <= 1e-4
    # only the ignored class present: the reference's mean([]) is the Python int 0
    only0 = torch.zeros(100, dtype=torch.long, device=dev)
    assert lovasz_softmax_flat(y[:100], only0, ignores=[0]) == 0
    # all rows left out: every per-class term is 0
    per = ops.LovaszClasses.apply(y[:100], torch.full((100,), -1, dtype=torch.int32, device=dev))
    assert float(per.abs().max()) == 0.0


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("case", ["no_targets", "no_valid_rows", "no_kept_query", "only_class_0"])
def test_degenerate_levels_match_the_original(ref, case):
    x = _scale_inputs(ref, N=20_000, Q=24, T=5, seed=2)
    if case == "no_targets":
        x["masks"], x["labels"] = x["masks"][:0], x["labels"][:0]
    elif case == "no_valid_rows":
        x["unknown"] = x["masks"].any(0, keepdim=True)
    elif case == "no_kept_query":
        x["ql"][..., K] += 50.0
    else:
        x["sem"] = torch.where(x["sem"] == 255, 255, 0).to(torch.uint8)
    crit = _criterion(ref, [x["cw"]], x["lw"])
    want = _one_level(ref, crit, x, False) if case != "no_targets" else None
    F = x["F"].clone()
    pred = {"voxel_logits": ref["ME"].SparseTensor(F, x["C"]), "query_logits": x["ql"]}
    target = [{"labels": x["labels"], "masks": x["masks"]}]
    z = torch.zeros(3, dtype=torch.long, device="cuda")
    got, falls = _run(ref, crit, pred, target, x["sem"], x["unknown"], 0, z, True)
    assert falls == []
    ref_ls, _ = _run(ref, crit, pred, target, x["sem"], x["unknown"], 0, z, False)
    for k in TERMS:
        a, b = got[k], ref_ls[k]
        assert type(a) is type(b) or (torch.is_tensor(a) and torch.is_tensor(b)), (k, type(a), type(b))
        va, vb = _val(a), _val(b)
        assert (np.isnan(va) and np.isnan(vb)) or abs(va - vb) <= 1e-4 * max(1.0, abs(vb)), (case, k, va, vb)
    if want is not None:
        print(case, want[0])


# ------------------------------------------------------------------------------------------------
# GPU: fallbacks, repeats, synchronisations
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("case", ["cpu", "bs2", "matcher", "classes", "outside", "no_labelled_row", "kept_over_128"])
def test_every_fallback_goes_to_the_original(ref, case):
    x = _scale_inputs(ref, N=5000, Q=150 if case == "kept_over_128" else 24, T=4, seed=4)
    if case == "no_labelled_row":
        x["sem"][:] = 255
    elif case == "kept_over_128":
        x["ql"][..., K] -= 50.0
    crit = _criterion(ref, [x["cw"]], x["lw"])
    pred = {"voxel_logits": ref["ME"].SparseTensor(x["F"], x["C"]), "query_logits": x["ql"]}
    target = [{"labels": x["labels"], "masks": x["masks"]}]
    min_C = torch.zeros(3, dtype=torch.long, device="cuda")
    sem, unknown = x["sem"], x["unknown"]
    if case == "cpu":
        pred = {"voxel_logits": type("R", (), {"F": x["F"].cpu(), "C": x["C"].cpu()})(), "query_logits": x["ql"].cpu()}
    elif case == "bs2":
        target = target * 2
    elif case == "matcher":
        class Other(ref["matcher"].HungarianMatcher):
            pass
        crit.matcher = Other(1.0, 20.0, 1.0)
    elif case == "classes":
        pred["query_logits"] = torch.randn(1, 24, 70, device="cuda")
    elif case == "outside":
        min_C = torch.tensor([0, 0, 8], device="cuda")
    from pasco_b200 import hooks
    cls = ref["cs"].SetCriterion
    calls = []
    orig = cls._pasco_b200_orig_compute_losses
    cls._pasco_b200_orig_compute_losses = lambda *a, **k: calls.append(1) or ("orig",)
    try:
        out = hooks._compute_losses(crit, None, pred, target, sem, unknown, 0, [], min_C)
    finally:
        cls._pasco_b200_orig_compute_losses = orig
    assert calls == [1] and out == ("orig",), case


def _compl_inputs(dev="cuda", C_=K, lo=0):
    """One subnet, scales 1 and 2: rows of a 16^3 box at lo, labels of a [16 / s]^3 volume."""
    g = torch.Generator().manual_seed(6)
    xyz = torch.nonzero(torch.rand(16, 16, 16, generator=g) < 0.3).int() + lo
    C = torch.cat([torch.zeros_like(xyz[:, :1]), xyz], 1).to(dev)
    sat = {s: [__import__("MinkowskiEngine").SparseTensor(torch.randn(C.shape[0], C_, generator=g).to(dev), C)]
           for s in (1, 2)}
    labels = {f"1_{s}": torch.randint(0, C_, (1, 16 // s, 16 // s, 16 // s), generator=g).to(torch.uint8).to(dev)
              for s in (1, 2)}
    freqs = {f"1_{s}": np.ones(C_) for s in (1, 2)}
    return labels, sat, [torch.zeros(3, dtype=torch.long)], [torch.full((3,), 15, dtype=torch.long)], freqs


def _spied_compl(fn, args):
    from pasco_b200 import hooks
    calls = []
    saved = hooks._orig_compl[:]
    hooks._orig_compl[:] = [lambda *a: calls.append(0) or ("orig",), lambda *a: calls.append(1) or ("orig",)]
    try:
        return fn(*args), calls
    finally:
        hooks._orig_compl[:] = saved


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("case", ["none", "cpu", "classes", "beyond", "no_present", "empty_kitti360"])
def test_completion_loss_fallbacks_go_to_the_original(ref, case):
    """Each input _sem_compl_loss leaves to the original, for the SemanticKITTI and the KITTI-360 loss."""
    from pasco_b200 import hooks
    labels, sat, mins, maxs, freqs = _compl_inputs(C_=70 if case == "classes" else K,
                                                   lo=100 if case == "empty_kitti360" else 0)
    if case == "cpu":
        sat[1] = [type("R", (), {"F": sat[1][0].F.cpu(), "C": sat[1][0].C.cpu()})()]
    elif case == "beyond":
        labels["1_1"] = labels["1_1"][:, :8].contiguous()
    elif case == "no_present":
        labels["1_2"][:] = 255
    for fn, which in ((hooks._compute_sem_compl_loss, 0), (hooks._compute_sem_compl_loss_kitti360, 1)):
        out, calls = _spied_compl(fn, (labels, sat, mins, maxs, freqs))
        if case == "none" or (case == "empty_kitti360" and which == 0):
            assert calls == [] and out != ("orig",), (case, which)       # the empty pairs are skipped: (0.0, 0.0)
            if case == "empty_kitti360":
                assert out == (0.0, 0.0)
        else:
            assert calls == [which] and out == ("orig",), (case, which, calls)


@pytest.mark.gpu
@needs_ref
def test_repeats_are_bit_identical_and_syncs_do_not_grow_with_n(ref):
    from pasco_b200 import hooks
    counts = {}
    for N in (50_000, 400_000):
        x = _scale_inputs(ref, N=N, seed=5)
        crit = _criterion(ref, [x["cw"]], x["lw"])
        outs = []
        for rep in range(2):
            F = x["F"].clone().requires_grad_(True)
            pred = {"voxel_logits": ref["ME"].SparseTensor(F, x["C"]), "query_logits": x["ql"]}
            target = [{"labels": x["labels"], "masks": x["masks"]}]
            z = torch.zeros(3, dtype=torch.long, device="cuda")
            torch.cuda.synchronize()
            with warnings.catch_warnings(record=True) as w:
                warnings.simplefilter("always")
                torch.cuda.set_sync_debug_mode("warn")
                try:
                    a, b = hooks._criterion_level(crit, pred, target, x["sem"], x["unknown"], 0, z)
                finally:
                    torch.cuda.set_sync_debug_mode("default")
            sites = collections.Counter(f"{os.path.basename(v.filename)}:{v.lineno}" for v in w
                                        if "called a synchronizing" in str(v.message))
            counts[N, rep] = sum(sites.values())
            vals = {**a, **b}
            total = sum(v for v in vals.values() if torch.is_tensor(v))
            total.backward()
            outs.append(({k: _val(v) for k, v in vals.items()}, F.grad.clone(), dict(sites)))
        assert outs[0][0] == outs[1][0], (N, outs[0][0], outs[1][0])
        assert torch.equal(outs[0][1], outs[1][1]), (N, float((outs[0][1] - outs[1][1]).abs().max()))
    print("synchronisations:", counts, outs[-1][2])
    assert len(set(counts.values())) == 1, counts
    assert set(counts.values()) <= set(range(hooks.CRITERION_SYNCS + 1)), outs[-1][2]
    # the completion loss over both scales: host bounds and label weights, one synchronisation per call
    args = _compl_inputs()
    hooks._compute_sem_compl_loss(*args)
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            out = hooks._compute_sem_compl_loss(*args)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    sites = [f"{os.path.basename(v.filename)}:{v.lineno}" for v in w if "called a synchronizing" in str(v.message)]
    assert torch.is_tensor(out[0]) and len(sites) <= hooks.CRITERION_SYNCS, sites


# ------------------------------------------------------------------------------------------------
# GPU: the unmodified Net end to end
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("M_", [1, 2])
def test_net_training_step_with_and_without_hook(ref, monkeypatch, M_):
    from pasco_b200 import hooks, ops
    from recipe import fill_state_dict
    ops.set_precision("fp32")
    hooks.uninstall()
    _, net = parity.reference_net(n_infers=M_)
    net.class_weights = [torch.ones(K + 1) for _ in range(M_)]
    net.criterion.class_weights = net.class_weights
    net.criterion.compl_labelweights = torch.ones(K)
    net.load_state_dict(fill_state_dict(net.state_dict()))
    net.object_mask_threshold = 0.05
    dev = torch.device("cuda")
    net.to(dev).train()
    meta = parity.INFER_MANIFEST["cases"]["m2" if M_ == 2 else "m1"]
    sc = parity.scene(meta, M_)
    grid = tuple(meta["grid"])
    g = torch.Generator().manual_seed(5)
    sem = torch.randint(0, K, (M_,) + grid, generator=g)
    sem[torch.rand(sem.shape, generator=g) < 0.6] = 0
    sem[:, :, :2, :] = 255
    mask_label = []
    for m in range(M_):
        present = [c for c in range(1, K) if (sem[m] == c).any()]
        mask_label.append({"labels": torch.tensor(present, dtype=torch.uint8, device=dev),
                           "masks": torch.stack([sem[m] == c for c in present]).to(dev)})
    batch = dict(in_feats=sc["in_feats"], in_coords=sc["in_coords"], min_Cs=[t.to(dev) for t in sc["min_Cs"]],
                 max_Cs=[t.to(dev) for t in sc["max_Cs"]], Ts=[t.to(dev) for t in sc["Ts"]],
                 global_min_Cs=sc["global_min_Cs"].to(dev), global_max_Cs=sc["global_max_Cs"].to(dev),
                 sem_labels=sc["sem_labels"], semantic_label=sem.to(torch.uint8).to(dev),
                 geo_labels={"1_1": torch.where(sem == 255, 255.0, (sem > 0).float()).to(dev)}, mask_label=mask_label)
    rec = _Assignments(ref, monkeypatch)

    def step():
        logged = {}
        net.log = lambda k, v, **kw: logged.__setitem__(k, _val(v))
        net.zero_grad(set_to_none=True)
        rec.got.clear()
        torch.manual_seed(0)
        out = net.step(batch, "train")
        out["loss"].backward()
        grads = {n: p.grad.detach().clone() for n, p in net.named_parameters() if p.grad is not None}
        return float(out["loss"]), logged, grads, [a for _, a in rec.got]

    want = step()
    again = step()                  # hooks off twice: what the network's own backward changes from run to run
    calls = []
    assert hooks.install(attention=False, criterion=True)
    cls = ref["cs"].SetCriterion
    orig = cls._pasco_b200_orig_compute_losses
    cls._pasco_b200_orig_compute_losses = lambda *a, **k: calls.append(1) or orig(*a, **k)
    saved = hooks._orig_compl[:]
    hooks._orig_compl[:] = [lambda *a: calls.append(2) or saved[0](*a), lambda *a: calls.append(3) or saved[1](*a)]
    try:
        got = step()
    finally:
        cls._pasco_b200_orig_compute_losses = orig
        hooks._orig_compl[:] = saved
    assert calls == [], "the hook fell back"
    assert len(got[3]) == len(want[3]) == 4 * M_
    for (qa, ta), (qb, tb) in zip(got[3], want[3]):
        assert np.array_equal(qa, qb) and np.array_equal(ta, tb), "assignments differ"
    assert set(got[1]) == set(want[1])
    for k, v in want[1].items():
        assert abs(got[1][k] - v) <= 1e-4 * max(1.0, abs(v)), (k, got[1][k], v)
    assert set(got[2]) == set(want[2])
    l2 = lambda a, b: float((a - b).double().norm() / b.double().norm().clamp(min=1e-30))  # noqa: E731
    err = {n: l2(got[2][n], want[2][n]) for n in want[2]}
    noise = {n: l2(again[2][n], want[2][n]) for n in want[2]}
    worst = sorted(err, key=err.get)[-5:]
    print(f"M = {M_}: loss {got[0]:.6f} vs {want[0]:.6f}; worst parameter-gradient relative L2 (hook on vs off, "
          f"off vs off): {[(n, f'{err[n]:.1e}', f'{noise[n]:.1e}') for n in worst]}")
    # parameters whose gradient the network's own backward reproduces: within 1e-3; the others (nondeterministic
    # reductions upstream of the criterion) within twice their run-to-run difference
    bad = {n: (err[n], noise[n]) for n in err if err[n] > max(1e-3, 2 * noise[n])}
    assert not bad, bad
