"""The evaluation hook (pasco_b200/hooks.py install(evaluate=True)): the unmodified reference's Net.evaluate_all on the
dense passes of csrc/metrics.cu, against the reference's own saved original on the same inputs.

  * CPU: the new C-ABI symbols are declared and typed, install / uninstall restore
    evaluate_all on both Net modules, the reference's float32 pair IoU (Tensor.__rdiv__), no local memory in the new
    kernels;
  * GPU: the three eval.npz scenes (make_golden_eval's predictions and ground truth) with all M + 1 entries, with and
    without uncertainty, hooked against the original (the original's ECE is torchmetrics 1.4's, restated as in
    make_golden_eval) and against the fixture; the all-unknown scene, no kept segment, argmax ties and NaN, a cropped
    training frame, every fallback (spied), bit-identical repeats and host synchronisations independent of Q and of
    the segment counts; the unmodified Net's training step and test-time step_inference with and without the hook.
GPU tests skip when oracle/_ref is not staged.
"""
import collections
import json
import math
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
import make_golden_predict as GP  # noqa: E402
import parity  # noqa: E402

STAGED = os.path.isdir(os.path.join(parity.REF, "pasco"))
needs_ref = pytest.mark.skipif(not STAGED, reason="oracle/_ref not staged")
SIZE = (256, 256, 32)
K = 20
FIX = np.load(os.path.join(HERE, "golden", "eval.npz"))
MANIFEST = json.load(open(os.path.join(HERE, "golden", "eval_manifest.json")))
NEW_SYMBOLS = ("pasco_eval_gt_volume", "pasco_eval_pairs_dense", "pasco_eval_ssc_planes", "pasco_eval_vox_dense")


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
    funcs = re.split(r"\n\s*Function : ", sass)
    names = ("k_eval_gt_volume", "k_eval_pairs_dense", "k_eval_ssc_planes", "k_eval_vox_dense")
    found = collections.Counter()
    for f in funcs:
        head = f.split("\n")[0]
        for n in names:
            if n in head:
                found[n] += 1
                assert not re.search(r"\b(LDL|STL)\b", f), f"{head}: local-memory traffic"
    assert set(found) == set(names) and found["k_eval_ssc_planes"] == 2 and found["k_eval_pairs_dense"] == 2


def test_reference_pair_iou_is_reciprocal_times_intersection():
    """The reference divides an np.int64 intersection by a 0-d torch area: Tensor.__rdiv__, reciprocal() * other."""
    from pasco_b200 import hooks
    g = np.random.default_rng(0)
    for _ in range(2000):
        union = int(g.integers(1, 400000))
        inter = int(g.integers(1, union + 1))
        want = np.int64(inter) / torch.tensor(union, dtype=torch.int64)
        assert want.dtype == torch.float32
        got = hooks._ref_iou(inter, union)
        assert isinstance(got, np.float32) and np.float32(float(want)) == got, (inter, union)


def _reference_modules():
    parity.reference_net()
    import importlib
    nps = importlib.import_module("pasco.models.net_panoptic_sparse")
    try:
        k360 = importlib.import_module("pasco.models.net_panoptic_sparse_kitti360")
    except Exception:
        k360 = None
    return nps, k360


@needs_ref
def test_install_uninstall_restores_evaluate_all():
    from pasco_b200 import hooks
    nps, k360 = _reference_modules()
    assert k360 is not None, "the KITTI-360 Net module is importable in the staged reference"
    before = (nps.Net.evaluate_all, k360.Net_kitti360.evaluate_all)
    assert hooks.install(attention=False)
    assert nps.Net.evaluate_all is before[0]                       # not requested: untouched
    for _ in range(2):
        assert hooks.install(attention=False, evaluate=True)
    assert nps.Net.evaluate_all is hooks._evaluate_all and k360.Net_kitti360.evaluate_all is hooks._evaluate_all_kitti360
    assert nps.Net._pasco_b200_orig_evaluate_all is before[0] and k360.Net_kitti360._pasco_b200_orig_evaluate_all is before[1]
    for _ in range(2):
        hooks.uninstall()
    assert (nps.Net.evaluate_all, k360.Net_kitti360.evaluate_all) == before


# ------------------------------------------------------------------------------------------------
# GPU: inputs
# ------------------------------------------------------------------------------------------------
@pytest.fixture
def ref(monkeypatch):
    """The reference with the post-processing hooks (the predictions' producer, checked against its originals by
    test_hooks_postprocess) and torchmetrics 1.4's calibration error in its metrics module."""
    from pasco_b200 import hooks, ops
    ops.set_precision("fp32")
    nps, k360 = _reference_modules()
    import MinkowskiEngine as ME
    from pasco.models import ensembler, helper, metrics as MET
    monkeypatch.setattr(MET, "binary_calibration_error", GE.binary_calibration_error)
    assert hooks.install(attention=False, postprocess=True)
    try:
        yield types.SimpleNamespace(ME=ME, ensembler=ensembler, helper=helper, MET=MET, nps=nps, k360=k360)
    finally:
        hooks.uninstall()


def _scene(r, seed, M=3, Q=GP.Q_A, labels_on_device=False):
    """make_golden_eval's scene `seed` on the device: ([(panop_out, sem_prob)] for the M + 1 entries, semantic label
    [1, X, Y, Z], mask label)."""
    preds, sems, Ts = GP.scene_a(seed=seed, M=M, Q=Q)
    bc = lambda c: torch.cat([torch.zeros_like(c[:, :1]), c], 1).int().cuda()  # noqa: E731
    Ts = [T.cuda() for T in Ts[:M]]
    ens = r.ensembler.Ensembler()
    sem_denses = ens.ensemble_sem_compl({1: [r.ME.SparseTensor(f.cuda(), bc(c)) for f, c in sems[:M]]}, Ts)
    ref_preds = [{"voxel_logits": r.ME.SparseTensor(p["voxel_logits"][0].cuda(), bc(p["voxel_logits"][1])),
                  "query_logits": p["query_logits"].cuda()} for p in preds[:M]]
    out = ens.ensemble_panop(ref_preds, sem_denses, SIZE, Ts, iou_threshold=GP.THR_A["iou_threshold"])
    entries = []
    for o, sd in zip(out, sem_denses):
        po = r.helper.panoptic_inference(o["voxel_probs"], o["query_probs"],
                                         overlap_threshold=GP.THR_A["overlap_threshold"],
                                         object_mask_threshold=GP.THR_A["object_mask_threshold"], thing_ids=GP.THING_IDS,
                                         min_C=torch.tensor([0, 0, 0]), scene_size=SIZE, input_query_logit=False,
                                         input_voxel_logit=False)
        entries.append((po, sd))
    sem, ml = GE.gt_scene(seed)
    labels = ml["labels"].cuda() if labels_on_device else ml["labels"]
    return entries, sem.unsqueeze(0).cuda(), {"labels": labels, "masks": ml["masks"].cuda()}


def _stub(r, n_entries, kitti=False, thresholds=(0.5,)):
    """make_golden_eval's stand-in for Net: what evaluate_all / evaluate_panoptic read from self."""
    Net = r.k360.Net_kitti360 if kitti else r.nps.Net
    s = types.SimpleNamespace(thing_ids=GP.THING_IDS, n_classes=K, uncertainty_thresholds=list(thresholds), sync_dist=False)
    s.uncertainty_metrics_by_thresholds = {t: {i: r.MET.UncertaintyMetrics() for i in range(n_entries)}
                                           for t in thresholds}
    s.evaluate_panoptic = types.MethodType(Net.evaluate_panoptic, s)
    s.panoptic_metrics = types.MethodType(Net.panoptic_metrics, s)
    s.log = lambda *a, **k: None
    s.orig = Net.evaluate_all                      # the unbound original (the hook is not installed on the class)
    s.fallbacks = []                               # the hook's calls of the saved original
    bound = types.MethodType(Net.evaluate_all, s)
    s._pasco_b200_orig_evaluate_all = lambda **kw: s.fallbacks.append(1) or bound(**kw)
    return s


def _metrics(r, n):
    from pasco.loss.panoptic_quality import PQStat
    return [PQStat() for _ in range(n)], [r.MET.SSCMetrics(K) for _ in range(n)]


def _copy_out(po):
    """The entry's panop_out with its own segment dicts (evaluate_panoptic records an "area" in them)."""
    return dict(po, segments_infos=[[dict(s) for s in po["segments_infos"][0]]])


def _call(r, stub, hooked, i, po, sd, sem, ml, pq, ssc, unc, kitti=False):
    from pasco_b200 import hooks
    kw = dict(ssc_confidence=sd.max(dim=0)[0], i_infer=i, sem_prob=sd, panop_out=po, semantic_label=sem,
              mask_labels=[ml], ssc_metrics=ssc, pq_stat=pq, uncertainty_metrics=r.MET.UncertaintyMetrics(),
              compute_uncertainty=unc)
    if hooked:
        return (hooks._evaluate_all_kitti360 if kitti else hooks._evaluate_all)(stub, **kw)
    return stub.orig(stub, **kw)


# ------------------------------------------------------------------------------------------------
# comparisons
# ------------------------------------------------------------------------------------------------
def _same_pq(a, b):
    assert list(a.pq_per_cat) == list(b.pq_per_cat), "categories touched in another order"
    for c in a.pq_per_cat:
        x, y = a.pq_per_cat[c], b.pq_per_cat[c]
        for f in ("tp", "fp", "fn", "all_n"):
            assert getattr(x, f) == getattr(y, f) and type(getattr(x, f)) is type(getattr(y, f)), (c, f)
        for f in ("iou", "all_iou"):
            u, v = getattr(x, f), getattr(y, f)
            assert torch.is_tensor(u) == torch.is_tensor(v), (c, f, u, v)
            if torch.is_tensor(u):
                assert u.dtype == v.dtype == torch.float32 and u.shape == v.shape and u.device == v.device, (c, f)
                assert np.float32(u.item()) == np.float32(v.item()), (c, f, u.item(), v.item())
            else:
                assert u == v and type(u) is type(v), (c, f)


def _close(a, b, atol=0.0, rtol=0.0):
    if math.isnan(a) or math.isnan(b):
        return math.isnan(a) and math.isnan(b)
    return abs(a - b) <= atol + rtol * abs(b)


def _same_ssc(a, b, unc, ece_atol=1e-6):
    """ece_atol: the original sums the calibration bins in fp32 (torchmetrics' scatter_add); over a full scene with
    millions of predicted non-empty cells that sum drifts by more than 1e-6 from the hook's double sums."""
    assert (a.completion_tp, a.completion_fp, a.completion_fn) == (b.completion_tp, b.completion_fp, b.completion_fn)
    for f in ("tps", "fps", "fns"):
        assert getattr(a, f).dtype == getattr(b, f).dtype and np.array_equal(getattr(a, f), getattr(b, f)), f
    if unc:
        for f in ("empty_ece", "nonempty_ece"):
            assert _close(getattr(a, f), getattr(b, f), atol=ece_atol), (f, getattr(a, f), getattr(b, f))
        for f in ("empty_nll", "nonempty_nll"):
            assert _close(getattr(a, f), getattr(b, f), rtol=1e-5), (f, getattr(a, f), getattr(b, f))
    for f in ("n_empty_voxels", "n_nonempty_voxels", "ece_count", "inference_time"):
        assert getattr(a, f) == getattr(b, f), f


def _same_unc(a, b):
    assert a.ins_confs == b.ins_confs and a.ins_correct == b.ins_correct and a.ins_sem_labels == b.ins_sem_labels
    assert [type(v) for v in a.ins_correct] == [type(v) for v in b.ins_correct]
    assert len(a.ins_all_class_probs) == len(b.ins_all_class_probs)
    assert all(torch.equal(x, y) for x, y in zip(a.ins_all_class_probs, b.ins_all_class_probs))
    assert _close(a.mask_ece, b.mask_ece, atol=1e-6), (a.mask_ece, b.mask_ece)
    for f in ("mask_auprc", "mask_auroc", "mask_fpr95", "mask_nll", "count"):
        assert getattr(a, f) == getattr(b, f), f


def _same_returns(a, b):
    (gs_a, gi_a, sp_a), (gs_b, gi_b, sp_b) = a, b
    for x, y in ((gs_a, gs_b), (sp_a, sp_b)):
        assert isinstance(x, np.ndarray) and x.dtype == y.dtype and x.shape == y.shape and np.array_equal(x, y)
    assert len(gi_a) == len(gi_b)
    for x, y in zip(gi_a, gi_b):
        assert set(x) == set(y)
        for k in ("id", "isthing", "category_id"):
            assert x[k] == y[k] and type(x[k]) is type(y[k]), k
        assert x["area"].dtype == y["area"].dtype and x["area"].shape == y["area"].shape == ()
        assert x["area"].device == y["area"].device and torch.equal(x["area"], y["area"])


def _same_segments(a, b):
    for x, y in zip(a["segments_infos"][0], b["segments_infos"][0]):
        assert ("area" in x) == ("area" in y)
        if "area" in x:
            assert x["area"] == y["area"] and type(x["area"]) is type(y["area"])


# ------------------------------------------------------------------------------------------------
# GPU: the fixture scenes
# ------------------------------------------------------------------------------------------------
def _run_scenes(r, unc, kitti=False):
    """Every fixture scene and entry through the hooked and the original evaluate_all (fresh and accumulated metrics):
    (per-scene hooked metrics, accumulated hooked (pq, ssc, stub), accumulated original (pq, ssc, stub))."""
    n = 4
    hs, os_ = _stub(r, n, kitti), _stub(r, n, kitti)
    tot_h, tot_o = _metrics(r, n), _metrics(r, n)
    per_scene = []
    for s_i, seed in enumerate(GE.SEEDS):
        entries, sem, ml = _scene(r, seed)
        one = _stub(r, n, kitti)
        for i, (po, sd) in enumerate(entries):
            pa, pb = _copy_out(po), _copy_out(po)
            got = _call(r, hs, True, i, pa, sd, sem, ml, tot_h[0][i], tot_h[1][i], unc, kitti)
            want = _call(r, os_, False, i, pb, sd, sem, ml, tot_o[0][i], tot_o[1][i], unc, kitti)
            _same_returns(got, want)
            _same_segments(pa, pb)
            _same_pq(tot_h[0][i], tot_o[0][i])
            _same_ssc(tot_h[1][i], tot_o[1][i], unc)
            _same_unc(hs.uncertainty_metrics_by_thresholds[0.5][i], os_.uncertainty_metrics_by_thresholds[0.5][i])
            pq1, ssc1 = _metrics(r, 1)
            _call(r, one, True, i, _copy_out(po), sd, sem, ml, pq1[0], ssc1[0], unc, kitti)
            per_scene.append((s_i, i, pq1[0], ssc1[0], one.uncertainty_metrics_by_thresholds[0.5][i]))
        assert one.fallbacks == [], f"scene {seed}: the hook fell back"
    assert hs.fallbacks == [], "the hook fell back"
    return per_scene, (tot_h[0], tot_h[1], hs), (tot_o[0], tot_o[1], os_)


def _check_against_fixture(per_scene, unc):
    for s_i, i, pq, ssc, um in per_scene:
        tag = f"s{s_i}e{i}"
        cats = sorted(pq.pq_per_cat)
        assert cats == FIX[tag + "_pq_cats"].tolist(), tag
        fields = np.array([[float(pq[c].all_iou), float(pq[c].all_n), float(pq[c].iou), pq[c].tp, pq[c].fp, pq[c].fn]
                           for c in cats], np.float64).reshape(-1, 6)
        np.testing.assert_allclose(fields, FIX[tag + "_pq_fields"], rtol=1e-6, atol=0, err_msg=tag)
        assert [ssc.completion_tp, ssc.completion_fp, ssc.completion_fn] == FIX[tag + "_completion"].tolist(), tag
        assert np.array_equal(np.stack([ssc.tps, ssc.fps, ssc.fns]).astype(np.int64), FIX[tag + "_class_counts"]), tag
        if unc:
            want = FIX[tag + "_ssc_unc"]
            got = [ssc.empty_ece, ssc.nonempty_ece, ssc.empty_nll, ssc.nonempty_nll, ssc.n_empty_voxels,
                   ssc.n_nonempty_voxels]
            for j, (a, b) in enumerate(zip(got, want)):
                assert _close(a, float(b), atol=1e-6 if j < 2 else 0, rtol=0 if j < 2 else 1e-5), (tag, j, a, b)
            assert _close(um.mask_ece, float(FIX[tag + "_mask_ece"][0]), atol=1e-6), tag


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("unc", [True, False])
def test_fixture_scenes_hooked_vs_original(ref, unc):
    per_scene, (pq_h, ssc_h, hs), (pq_o, ssc_o, os_) = _run_scenes(ref, unc)
    _check_against_fixture(per_scene, unc)
    for i in range(4):
        fin = MANIFEST["final"][i]
        d = ssc_h[i].get_stats()
        for k in ("precision", "recall", "iou", "iou_ssc_mean"):
            assert _close(float(d[k]), fin[k], rtol=1e-9), (i, k)
        pm = hs.panoptic_metrics(pq_h[i])
        pm_o = os_.panoptic_metrics(pq_o[i])
        for name in ("All", "Things", "Stuff"):
            for k, v in pm[name].items():
                assert float(v) == float(pm_o[name][k]), (i, name, k)
                assert _close(float(v), fin[name][k], rtol=1e-6), (i, name, k)
        if unc:
            for k in ("empty_ece", "nonempty_ece"):
                assert _close(float(d[k]), fin[k], atol=1e-6), (i, k)
            for k in ("empty_nll", "nonempty_nll"):
                assert _close(float(d[k]), fin[k], rtol=1e-5), (i, k)
            u = hs.uncertainty_metrics_by_thresholds[0.5][i].get_stats()
            u_o = os_.uncertainty_metrics_by_thresholds[0.5][i].get_stats()
            for k in ("mask_ece", "ins_ece", "ins_nll", "count"):
                assert _close(float(u[k]), float(u_o[k]), atol=1e-6), (i, k)
                assert _close(float(u[k]), fin[k], atol=1e-6), (i, k)


@pytest.mark.gpu
@needs_ref
def test_kitti360_net_hooked_vs_original(ref):
    assert ref.k360 is not None
    _run_scenes(ref, True, kitti=True)


# ------------------------------------------------------------------------------------------------
# GPU: edge cases and fallbacks
# ------------------------------------------------------------------------------------------------
def _both(r, po, sd, sem, ml, unc=True, conf=None, i=0):
    """One call of each on fresh metrics, compared field by field."""
    hs, os_ = _stub(r, 1), _stub(r, 1)
    (pq_h,), (ssc_h,) = _metrics(r, 1)
    (pq_o,), (ssc_o,) = _metrics(r, 1)
    from pasco_b200 import hooks
    pa, pb = _copy_out(po), _copy_out(po)
    c = sd.max(dim=0)[0] if conf is None else conf
    kw = dict(ssc_confidence=c, i_infer=i, sem_prob=sd, semantic_label=sem, mask_labels=[ml],
              uncertainty_metrics=r.MET.UncertaintyMetrics(), compute_uncertainty=unc)
    got = hooks._evaluate_all(hs, panop_out=pa, ssc_metrics=ssc_h, pq_stat=pq_h, **kw)
    want = os_.orig(os_, panop_out=pb, ssc_metrics=ssc_o, pq_stat=pq_o, **kw)
    assert hs.fallbacks == [], "the hook fell back"
    _same_returns(got, want)
    _same_segments(pa, pb)
    _same_pq(pq_h, pq_o)
    _same_ssc(ssc_h, ssc_o, unc)
    _same_unc(hs.uncertainty_metrics_by_thresholds[0.5][i], os_.uncertainty_metrics_by_thresholds[0.5][i])
    return got, pq_h, ssc_h


@pytest.mark.gpu
@needs_ref
def test_edge_cases(ref):
    entries, sem, ml = _scene(ref, 0, M=1)
    po, sd = entries[0]
    # the all-unknown scene
    _both(ref, po, sd, torch.full_like(sem, 255), ml)
    # no kept segment: every predicted id zeroed, no segment records
    empty = dict(po, panoptic_seg_denses=torch.zeros_like(po["panoptic_seg_denses"]), segments_infos=[[]])
    _both(ref, empty, sd, sem, ml)
    # argmax ties and NaN in the class planes (the given confidence stays finite)
    sd2 = sd.clone()
    known = (sem[0] != 255) & (sem[0] == 0)
    idx = torch.nonzero(known.reshape(-1))[:, 0]
    sel = idx[::5]                                            # four disjoint cell sets
    tie, nan, nan2, nan3 = sel[0::4][:5000], sel[1::4][:3000], sel[2::4][:2000], sel[3::4][:2000]
    flat = sd2.view(K, -1)
    flat[5, tie] = flat[:, tie].max(0)[0]
    flat[3, tie] = flat[5, tie]
    flat[7, nan] = float("nan")
    # NaN in two or three planes: the first NaN wins
    flat[9, nan2] = float("nan")
    flat[4, nan2] = float("nan")
    flat[12, nan3] = float("nan")
    flat[2, nan3] = float("nan")
    flat[15, nan3] = float("nan")
    got, _, _ = _both(ref, po, sd2, sem, ml, conf=sd.max(dim=0)[0])
    pred = torch.from_numpy(got[2]).view(-1)
    assert bool((pred[nan.cpu()] == 7).all()) and bool((pred[nan2.cpu()] == 4).all())
    assert bool((pred[nan3.cpu()] == 2).all())
    for cells in (tie, nan, nan2, nan3):
        assert torch.equal(pred[cells.cpu()], torch.argmax(flat[:, cells], 0).cpu())
    # a cropped frame (a training subnet's box: not 256 x 256 x 32, not at the origin)
    box = (slice(40, 136), slice(60, 140), slice(8, 24))
    crop = lambda v: v[(slice(None),) + box].contiguous()  # noqa: E731
    po_c = dict(po, panoptic_seg_denses=crop(po["panoptic_seg_denses"]),
                vox_confidence_denses=crop(po["vox_confidence_denses"]),
                vox_all_mask_probs_denses=[po["vox_all_mask_probs_denses"][0]])
    ml_c = {"labels": ml["labels"], "masks": crop(ml["masks"])}
    got, pq, _ = _both(ref, po_c, crop(sd), crop(sem), ml_c)
    assert got[0].shape == (96, 80, 16) and got[2].shape == (1, 96, 80, 16)
    _both(ref, po_c, crop(sd), crop(sem), ml_c, unc=False)


@pytest.mark.gpu
@needs_ref
def test_fallbacks_reach_the_original(ref):
    from pasco_b200 import hooks
    entries, sem, ml = _scene(ref, 0, M=1)
    po, sd = entries[0]
    calls = []

    def reaches_original(po=po, sd=sd, sem=sem, ml=ml, thresholds=(0.5,), ssc_k=K):
        s = _stub(ref, 1, thresholds=thresholds)
        s._pasco_b200_orig_evaluate_all = lambda **kw: calls.append(1)
        n = len(calls)
        (pq,), _ = _metrics(ref, 1)
        hooks._evaluate_all(s, ssc_confidence=sd.max(dim=0)[0], i_infer=0, sem_prob=sd, panop_out=_copy_out(po),
                            semantic_label=sem, mask_labels=[ml], ssc_metrics=ref.MET.SSCMetrics(ssc_k), pq_stat=pq,
                            uncertainty_metrics=None, compute_uncertainty=True)
        assert pq.pq_per_cat == {}, "a fallback left the metrics touched"
        return len(calls) == n + 1

    assert reaches_original(sd=sd.cpu())                                                          # CPU tensors
    wide = torch.softmax(torch.randn((70,) + SIZE, device="cuda"), 0)
    assert reaches_original(sd=wide, ssc_k=70)                                                    # K > 64
    assert reaches_original(po=dict(po, panoptic_seg_denses=po["panoptic_seg_denses"].repeat(2, 1, 1, 1)))  # 2 items
    assert reaches_original(thresholds=(0.2, 0.5))                                                # Hungarian branch
    assert reaches_original(sem=sem[:, :128])                                                     # shapes disagree
    bad = sem.clone()
    bad[0, 3, 3, 3] = 30
    assert reaches_original(sem=bad)                                                              # label >= K
    assert reaches_original(ml=dict(ml, labels=torch.cat([ml["labels"], torch.tensor([40])]),
                                    masks=torch.cat([ml["masks"], ml["masks"][:1]])))             # mask class >= K
    pan = po["panoptic_seg_denses"].clone()
    pan[0, 100, 100, 10] = 999
    if sem[0, 100, 100, 10] == 255:
        sem = sem.clone()
        sem[0, 100, 100, 10] = 0
    assert reaches_original(po=dict(po, panoptic_seg_denses=pan), sem=sem)                        # id without a segment
    assert len(calls) == 8


@pytest.mark.gpu
@needs_ref
def test_repeat_calls_bit_identical(ref):
    entries, sem, ml = _scene(ref, 1, M=1)
    po, sd = entries[-1]
    runs = []
    for _ in range(2):
        got, pq, ssc = _both(ref, po, sd, sem, ml)
        runs.append((got, pq, ssc))
    (a, pa, sa), (b, pb, sb) = runs
    _same_returns(a, b)
    _same_pq(pa, pb)
    for f in ("empty_ece", "nonempty_ece", "empty_nll", "nonempty_nll"):
        x, y = getattr(sa, f), getattr(sb, f)
        assert x == y or (math.isnan(x) and math.isnan(y)), f


@pytest.mark.gpu
@needs_ref
def test_host_synchronisations_are_constant(ref):
    from pasco_b200 import hooks
    counts = {}
    entries, sem, ml = _scene(ref, 0, M=1, labels_on_device=True)
    (pq,), (ssc,) = _metrics(ref, 1)
    hooks._evaluate_all(_stub(ref, 2), ssc_confidence=entries[0][1].max(dim=0)[0], i_infer=0, sem_prob=entries[0][1],
                        panop_out=_copy_out(entries[0][0]), semantic_label=sem, mask_labels=[ml], ssc_metrics=ssc,
                        pq_stat=pq, uncertainty_metrics=None, compute_uncertainty=True)      # first use of pinned memory
    for Q in (24, 100, 200):
        entries, sem, ml = _scene(ref, 0, M=1, Q=Q, labels_on_device=True)
        for i, (po, sd) in enumerate(entries):
            for unc in (True, False):
                s = _stub(ref, 2)
                (pq,), (ssc,) = _metrics(ref, 1)
                conf = sd.max(dim=0)[0]
                torch.cuda.synchronize()
                with warnings.catch_warnings(record=True) as w:
                    warnings.simplefilter("always")
                    torch.cuda.set_sync_debug_mode("warn")
                    try:
                        hooks._evaluate_all(s, ssc_confidence=conf, i_infer=i, sem_prob=sd, panop_out=_copy_out(po),
                                            semantic_label=sem, mask_labels=[ml], ssc_metrics=ssc, pq_stat=pq,
                                            uncertainty_metrics=None, compute_uncertainty=unc)
                    finally:
                        torch.cuda.set_sync_debug_mode("default")
                sites = collections.Counter(f"{os.path.basename(x.filename)}:{x.lineno}" for x in w
                                            if "synchroniz" in str(x.message)
                                            and f"{os.sep}pasco_b200{os.sep}" in x.filename)
                counts[Q, i, unc] = (sum(sites.values()), len(po["segments_infos"][0]))
                print(f"Q = {Q}, entry {i}, uncertainty {unc}: {dict(sites)}")
    segs = {v[1] for v in counts.values()}
    assert len(segs) > 1, "the segment counts differ between the cases"
    assert {v[0] for k, v in counts.items() if k[2]} == {hooks.EVAL_SYNCS}
    assert {v[0] for k, v in counts.items() if not k[2]} == {hooks.EVAL_SYNCS - 1}


# ------------------------------------------------------------------------------------------------
# GPU: the unmodified Net end to end
# ------------------------------------------------------------------------------------------------
def _net_metrics(net, step):
    out = {}
    for i in net.pq_stat[step]:
        out[i] = (net.pq_stat[step][i], net.ssc_metrics[step][i], net.uncertainty_metrics_by_thresholds[0.5][i])
    return out


def _fresh(net, step):
    from pasco.loss.panoptic_quality import PQStat
    from pasco.models.metrics import SSCMetrics, UncertaintyMetrics
    for i in net.pq_stat[step]:
        net.pq_stat[step][i] = PQStat()
        net.ssc_metrics[step][i] = SSCMetrics(net.n_classes)
        net.uncertainty_metrics[step][i] = UncertaintyMetrics()
        net.uncertainty_metrics_by_thresholds[0.5][i] = UncertaintyMetrics()


def _same_net_metrics(a, b, unc):
    assert set(a) == set(b)
    for i in a:
        _same_pq(a[i][0], b[i][0])
        _same_ssc(a[i][1], b[i][1], unc, ece_atol=1e-4)
        _same_unc(a[i][2], b[i][2])


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("M", [1, 2])
def test_net_training_step_with_and_without_hook(ref, M):
    """Net.step(batch, "train"): evaluate_all on subnets 0 and M − 1 in their own frames.  Same loss, same metrics."""
    from pasco_b200 import hooks
    from recipe import fill_state_dict
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

    def step():
        _fresh(net, "train")
        torch.manual_seed(0)
        out = net.step(batch, "train")
        return out, _net_metrics(net, "train")

    want, want_m = step()
    calls = []
    assert hooks.install(attention=False, evaluate=True)
    try:
        orig = ref.nps.Net._pasco_b200_orig_evaluate_all
        ref.nps.Net._pasco_b200_orig_evaluate_all = lambda *a, **k: calls.append(1) or orig(*a, **k)
        got, got_m = step()
    finally:
        ref.nps.Net._pasco_b200_orig_evaluate_all = orig
        hooks.uninstall()
    assert torch.equal(got["loss"], want["loss"])
    assert calls == [], "the hook fell back"
    print("training frames:", [tuple(p["panoptic_seg_denses"].shape) for p in got["panop_out_subnets"]])
    _same_net_metrics(got_m, want_m, False)


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("M", [1, 3])
def test_net_step_inference_with_and_without_hook(ref, M, capsys):
    """Net.step_inference(batch, "test", eval=True) for all M + 1 entries, then test_epoch_end's tables."""
    from pasco_b200 import hooks
    ME, net = parity.reference_net(n_infers=M)
    if M == 1:
        net, _ = parity.load_eval(net, "m1", ref_names=False)
    else:
        from recipe import fill_state_dict
        net.load_state_dict(fill_state_dict(net.state_dict()))
        net.cuda().eval()
    net.object_mask_threshold = 0.05
    dev = torch.device("cuda")
    meta = parity.INFER_MANIFEST["cases"]["m1"]
    sc = parity.scene(meta, M)
    sem, ml = GE.gt_scene(0)
    ml = {"labels": ml["labels"].to(dev), "masks": ml["masks"].to(dev)}
    batch = dict(in_feats=sc["in_feats"], in_coords=sc["in_coords"], min_Cs=[t.to(dev) for t in sc["min_Cs"]],
                 max_Cs=[t.to(dev) for t in sc["max_Cs"]], Ts=[t.to(dev) for t in sc["Ts"]],
                 global_min_Cs=sc["global_min_Cs"].to(dev), global_max_Cs=sc["global_max_Cs"].to(dev),
                 geo_labels=sc["sem_labels"], mask_classes=sc["mask_classes"],
                 semantic_label=sem.unsqueeze(0).to(dev), semantic_label_origin=sem.unsqueeze(0).to(dev),
                 mask_label=[ml], mask_label_origin=[ml])

    def run():
        _fresh(net, "test")
        with torch.no_grad():
            out = net.step_inference(batch, "test", eval=True)
        capsys.readouterr()
        net.test_epoch_end([])
        return out, _net_metrics(net, "test"), capsys.readouterr().out

    want, want_m, want_t = run()
    calls = []
    assert hooks.install(attention=False, evaluate=True)
    try:
        orig = ref.nps.Net._pasco_b200_orig_evaluate_all
        ref.nps.Net._pasco_b200_orig_evaluate_all = lambda *a, **k: calls.append(1) or orig(*a, **k)
        got, got_m, got_t = run()
    finally:
        ref.nps.Net._pasco_b200_orig_evaluate_all = orig
        hooks.uninstall()
    assert calls == [], "the hook fell back"
    _same_net_metrics(got_m, want_m, True)
    for a, b in zip(zip(*got[1:]), zip(*want[1:])):
        _same_returns(a, b)
    assert got_t == want_t and "ensemble" in got_t
