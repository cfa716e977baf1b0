"""metrics.Evaluator and its counting passes (csrc/metrics.cu) against a dense torch restatement of the reference's
evaluation (Net.evaluate_all with pq_compute_single_core, find_matched_segment, SSCMetrics and UncertaintyMetrics) and
against a fixture the reference's own code produced (tests/golden/make_golden_eval.py).

  * CPU: the new entry points' header and ctypes signatures; the torchmetrics 1.4 restatement against hand-computed
    bins (a confidence of 1.0 in its own slot, NaN for an empty input); the ECE from bins; the ground-truth walk; the
    host finishing fed by the torch restatement of the counting passes on the torch post-processing (ensemble.py) of
    the rebuilt fixture inputs, against the fixture and its printed tables;
  * GPU: the per-scene tables (PQ fields, matches, SSC counts, ECE / NLL), the final dicts and the printed tables
    against the fixture; every kernel table (ground truth, pairs, confusion, calibration bins, NLL and confidence sums,
    voxel bins) against the restatement at Q = 100, 200 and 600, integers exactly and sums to 1e-6; confidences on the
    exact fp32 slot boundaries and 1.0; a pair table too large for shared memory; PascoNet.predict(keep_sem_rows=True)
    end to end against the restatement fed by ensemble.py; an all-unknown scene; bit-identical repeat calls; host
    synchronisations independent of Q and G; input validation, including entries predicted on a larger grid than the
    ground truth, which must leave the accumulated metrics unchanged.
"""
import json
import math
import os
import sys
import warnings

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLD = os.path.join(HERE, "golden")
sys.path.insert(0, ROOT)
sys.path.insert(0, GOLD)
import make_golden_eval as GE  # noqa: E402  (gt_scene rebuilds the fixture's ground truth; the reference is not imported)
import make_golden_predict as GP  # noqa: E402
import parity  # noqa: E402

from pasco_b200 import metrics as MT  # noqa: E402

FIX = np.load(os.path.join(GOLD, "eval.npz"))
MANIFEST = json.load(open(os.path.join(GOLD, "eval_manifest.json")))
K = 20


def _rel(a, b, tol=1e-6, atol=0.0):
    if isinstance(a, float) and math.isnan(a):
        return isinstance(b, float) and math.isnan(b)
    return abs(a - b) <= max(tol * max(abs(a), abs(b), 1e-12), atol)


# An ECE lies in [0, 1] and the reference's is a float32 result of float32 slot sums over up to 2 M confidences, while
# the device sums in double: compare at float32 resolution
ECE_ATOL = 1e-7


# ------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------
def test_calibration_error_bins():
    conf = torch.tensor([1.0, 0.5, 0.05, 1.0])
    correct = torch.tensor([True, False, True, False])
    # slots: 1.0 → 15 (its own), 0.5 → 7 (7/15 <= 0.5 < 8/15), 0.05 → 0
    want = (abs(0.5 - 1.0) * 2 + abs(0 - 0.5) + abs(1 - 0.05)) / 4
    assert abs(float(MT.calibration_error(conf, correct)) - want) < 1e-6
    cnt, sc, sk = np.zeros(16), np.zeros(16), np.zeros(16)
    for c, k in zip(conf.tolist(), correct.tolist()):
        s = int(torch.bucketize(torch.tensor([c]), torch.linspace(0, 1, 16), right=True)[0]) - 1
        cnt[s] += 1
        sc[s] += c
        sk[s] += k
    assert cnt[15] == 2 and cnt[7] == 1 and cnt[0] == 1
    assert abs(MT.ece_from_bins(cnt, sc, sk) - want) < 1e-7                 # 0.05 is not exact in fp32
    assert math.isnan(float(MT.calibration_error(torch.zeros(0), torch.zeros(0, dtype=torch.bool))))
    assert math.isnan(MT.ece_from_bins(np.zeros(16), np.zeros(16), np.zeros(16)))


def test_gt_walk():
    seg_of, segs = MT.gt_walk([0, 9, 1, 9, 1, 10], (1, 2))
    assert seg_of == [0, 1, 2, 1, 3, 4]
    assert segs == [(1, 9, False, 1), (2, 1, True, 2), (3, 1, True, 4), (4, 10, False, 5)]


def test_fixture_manifest():
    assert MANIFEST["seeds"] == list(GE.SEEDS) and MANIFEST["n_classes"] == K
    assert sorted(FIX.files) == MANIFEST["arrays"]
    kinds = [(c["n_pq_pairs"], c["n_matches"], c["n_pred_segments"]) for c in MANIFEST["cases"][0]["entries"]]
    assert all(k[0] > 0 and k[1] > 0 for k in kinds)
    assert all(e["n_pred_segments"] == 0 for e in MANIFEST["cases"][2]["entries"])


# ------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------
def _entries(seed=0, Q=GP.Q_A, M=3):
    from pasco_b200 import predict as P
    preds, sems, Ts = GP.scene_a(seed=seed, M=M, Q=Q)
    cu = lambda t: t.cuda()                                     # noqa: E731
    preds = [{"voxel_logits": tuple(map(cu, p["voxel_logits"])), "query_logits": cu(p["query_logits"])} for p in preds]
    sems = [tuple(map(cu, s)) for s in sems]
    return P.postprocess(preds, sems, Ts, keep_sem_rows=True, **GP.THR_A)


def _gt(seed):
    sem, ml = GE.gt_scene(seed)
    return sem.cuda(), {"labels": ml["labels"].cuda(), "masks": ml["masks"].cuda()}


BOUNDS = torch.linspace(0, 1, 16, dtype=torch.float32)


def _slot(conf):
    return (torch.bucketize(conf, BOUNDS.to(conf.device), right=True) - 1).clamp(min=0)


def r_gt(masks, seg_of, label, G, K):
    """Torch restatement of k_eval_gt: (gt id per cell, mask sums, id areas after zeroing, known-cell histogram)."""
    n, cells = masks.shape[0], label.numel()
    m = masks.reshape(n, cells)
    gt = torch.zeros(cells, dtype=torch.long, device=label.device)
    for i in range(n):
        if seg_of[i]:
            gt[m[i]] = seg_of[i]
    lab = label.reshape(-1).long()
    unk = lab == 255
    gt[unk] = 0
    hist = torch.bincount(lab[~unk].clamp(max=K), minlength=K + 1)
    return gt, m.sum(1).cpu().numpy(), torch.bincount(gt, minlength=G + 1).cpu().numpy(), hist.cpu().numpy()


def r_p_target(e, cells, target):
    """p[target] of the entry's averaged class distribution at the cells (the mean of the subnets' rows, an absent
    subnet one-hot class 0, summed in subnet order); a dense entry holds the distribution itself."""
    if "sem_dense" in e:
        return e["sem_dense"][target, cells]
    acc = torch.zeros(cells.shape[0], dtype=torch.float32, device=cells.device)
    for prob, cell_row in e["sem_rows"]:
        r = cell_row[cells].long()
        v = (target == 0).float()
        v[r >= 0] = prob[r[r >= 0], target[r >= 0]]
        acc = acc + v
    return acc / len(e["sem_rows"])


def r_entry(e, gt, label, G, S, K, nll=True):
    """Torch restatement of k_eval_pairs + k_eval_ssc, in _entry_tables' layout."""
    cells = label.numel()
    lab = label.reshape(-1).long()
    lin, pan = e["lin"].long(), e["panoptic_seg"].long()
    ok = (lin >= 0) & (lin < cells)
    bad = int((~ok).sum())
    lin, pan = lin[ok], pan[ok]
    sel = (pan != 0) & (lab[lin] != 255)
    out = sel & ((pan < 0) | (pan > S))
    sel &= ~out
    pairs = torch.bincount(gt[lin[sel]] * (S + 1) + pan[sel], minlength=(G + 1) * (S + 1)).view(G + 1, S + 1)
    pred_area = torch.bincount(pan[sel], minlength=S + 1)
    pred_area[0] = bad + int(out.sum())
    c = e["ssc_lin"].long()
    ok = (c >= 0) & (c < cells)
    sbad = int((~ok).sum())
    c, pr, cf = c[ok], e["ssc_pred"][ok].long(), e["ssc_confidence"][ok]
    known = lab[c] != 255
    c, pr, cf = c[known], pr[known], cf[known]
    t = lab[c]
    good = (pr >= 0) & (pr < K) & (t < K)
    sbad += int((~good).sum())
    c, pr, cf, t = c[good], pr[good], cf[good], t[good]
    idx = (pr != 0).long() * 16 + _slot(cf)
    cnt = torch.bincount(idx, minlength=32)
    cor = torch.bincount(idx[pr == t], minlength=32)
    sums = torch.zeros(34, dtype=torch.float64, device=c.device)
    sums[:32].index_add_(0, idx, cf.double())
    if nll:
        v = -torch.log(r_p_target(e, c, t) + 1e-12)
        sums[32:34].index_add_(0, (pr != 0).long(), v.double())
    cal = torch.stack([cnt.view(2, 16), cor.view(2, 16)], 1)
    return {"pairs": pairs.cpu().numpy(), "pred_area": pred_area.cpu().numpy(),
            "conf": torch.bincount(t * K + pr, minlength=K * K).view(K, K).cpu().numpy().astype(np.int64),
            "cal": cal.cpu().numpy().astype(np.int64), "bad": sbad, "sums": sums.cpu().numpy()}


def r_vox(e, gt, match):
    """Torch restatement of k_eval_vox: (cal [2, 16], confidence sums [16])."""
    cells = gt.numel()
    lin, pan, cf = e["lin"].long(), e["panoptic_seg"].long(), e["vox_confidence"]
    ok = (lin >= 0) & (lin < cells)
    lin, pan, cf = lin[ok], pan[ok], cf[ok]
    g = gt[lin]
    q = (cf != 0) & (g != 0)
    lin, pan, cf, g = lin[q], pan[q], cf[q], g[q]
    m = torch.as_tensor(match, device=gt.device).long()
    inside = (pan > 0) & (pan < m.numel())
    mapped = torch.zeros_like(pan)
    mapped[inside] = m[pan[inside]]
    slot = _slot(cf)
    cal = torch.stack([torch.bincount(slot, minlength=16), torch.bincount(slot[mapped == g], minlength=16)])
    sums = torch.zeros(16, dtype=torch.float64, device=gt.device).index_add_(0, slot, cf.double())
    return cal.cpu().numpy(), sums.cpu().numpy()


class RestatedEvaluator(MT.Evaluator):
    """The Evaluator's host finishing fed by the torch restatement of the counting passes, on any device."""

    def _gt_tables(self, masks, seg_of, label, G):
        return r_gt(masks, seg_of, label, G, self.K)

    def _entry_tables(self, e, gt_id, label, G, S):
        return r_entry(e, gt_id, label, G, S, self.K, nll=self.uncertainty)

    def _vox_tables(self, e, gt_id, match):
        return r_vox(e, gt_id, match)


def _torch_entries(preds, sems, Ts, thr=GP.THR_A, thing_ids=GP.THING_IDS):
    """ensemble.py's post-processing as Evaluator entries: panoptic rows, and the dense class distribution as one
    semantic row per cell (a cell without a row already holds one-hot class 0 there)."""
    from pasco_b200 import ensemble as E
    sem_denses = E.ensemble_sem_compl(sems, Ts)
    out = E.ensemble_panop(preds, sem_denses, Ts, iou_threshold=thr["iou_threshold"])
    entries = []
    for o, sd in zip(out, sem_denses):
        prob, lin = o["voxel_probs"]
        order = torch.argsort(lin)
        pan, _, conf, infos = E.panoptic_inference_with_confidence(prob[order], o["query_probs"][0],
                                                                   thr["overlap_threshold"], thr["object_mask_threshold"],
                                                                   thing_ids)
        flat = sd.reshape(sd.shape[0], -1)
        best, arg = flat.max(0)
        entries.append({"lin": lin[order].long(), "panoptic_seg": pan.int(), "vox_confidence": conf.float(),
                        "segments_info": infos, "ssc_lin": torch.arange(flat.shape[1], device=flat.device),
                        "ssc_pred": flat.argmax(0).int(), "ssc_confidence": best, "sem_dense": flat, "sem_rows": []})
    return entries


def _check_fixture(ev, entries_of, gt_of):
    for s_i, seed in enumerate(GE.SEEDS):
        ev.update(entries_of(seed), *gt_of(seed))
        for i, rec in enumerate(ev.last_scene):
            tag = f"s{s_i}e{i}"
            cats = FIX[tag + "_pq_cats"].tolist()
            assert sorted(rec["pq"]) == cats, tag
            for c, want in zip(cats, FIX[tag + "_pq_fields"]):
                got = rec["pq"][c]
                assert list(got[3:]) == [int(v) for v in want[3:]], (tag, c)
                assert got[1] == want[1] and _rel(got[0], want[0]) and _rel(got[2], want[2]), (tag, c, got, want)
            assert rec["pq_pairs"] == [tuple(p) for p in FIX[tag + "_pq_pairs"].tolist()], tag
            assert rec["matches"] == [tuple(p) for p in FIX[tag + "_matches"].tolist()], tag
            assert list(rec["completion"]) == FIX[tag + "_completion"].tolist(), tag
            np.testing.assert_array_equal(np.stack([rec["tps"], rec["fps"], rec["fns"]]), FIX[tag + "_class_counts"])
            eece, nece, enll, nnll, ne, nn = FIX[tag + "_ssc_unc"].tolist()
            assert _rel(rec["empty_ece"], eece, atol=ECE_ATOL) and _rel(rec["nonempty_ece"], nece, atol=ECE_ATOL), \
                (tag, rec["empty_ece"], eece, rec["nonempty_ece"], nece)
            assert _rel(rec["nll_sums"][0], enll) and _rel(rec["nll_sums"][1], nnll), (tag, rec["nll_sums"], enll, nnll)
            assert rec["n_voxels"] == (ne, nn), tag
            assert _rel(rec["mask_ece"], float(FIX[tag + "_mask_ece"][0]), atol=ECE_ATOL), (tag, rec["mask_ece"])
    for i, (got, want) in enumerate(zip(ev.compute(), MANIFEST["final"])):
        for k in ("precision", "recall", "iou", "iou_ssc_mean", "empty_ece", "nonempty_ece", "empty_nll",
                  "nonempty_nll", "mask_ece", "ins_ece", "ins_nll", "count"):
            assert _rel(float(got[k]), float(want[k]), 1e-6, ECE_ATOL if k.endswith("ece") else 0.0), (i, k, got[k],
                                                                                                       want[k])
        np.testing.assert_allclose(got["iou_ssc"], want["iou_ssc"], rtol=1e-6)
        for g in ("All", "Things", "Stuff"):
            for k in ("pq_dagger", "pq", "sq", "rq", "n") if g == "All" else ("pq", "sq", "rq", "n"):
                assert _rel(float(got[g][k]), float(want[g][k])), (i, g, k, got[g][k], want[g][k])
        assert sorted(map(str, got["per_class"])) == sorted(want["per_class"])
    assert ev.tables() == MANIFEST["tables"]


def test_host_finishing_on_restated_tables_matches_fixture():
    """The host finishing is fed by the torch restatement of the counting passes on ensemble.py's post-processing of
    the rebuilt fixture inputs, on the CPU."""
    def entries_of(seed):
        return _torch_entries(*GP.scene_a(seed=seed))

    def gt_of(seed):
        sem, ml = GE.gt_scene(seed)
        return sem, ml
    _check_fixture(RestatedEvaluator(4, K, GP.THING_IDS), entries_of, gt_of)


@pytest.mark.gpu
def test_fixture_scenes():
    _check_fixture(MT.Evaluator(4, K, GP.THING_IDS, uncertainty=True), _entries, _gt)


def _compare_tables(ev, entries, sem, ml):
    """Every device table of one scene against the restatement: integers exactly, double sums to 1e-6."""
    labels = [int(v) for v in ml["labels"].tolist()]
    seg_of, segs = MT.gt_walk(labels, ev.thing_ids)
    G = len(segs)
    label = sem.reshape(-1).to(torch.uint8).contiguous()
    gt_id, mask_sum, id_area, hist = ev._gt_tables(ml["masks"], seg_of, label, G)
    r_id, r_sum, r_area, r_hist = r_gt(ml["masks"], seg_of, label, G, K)
    assert torch.equal(gt_id.long(), r_id)
    np.testing.assert_array_equal(mask_sum, r_sum)
    np.testing.assert_array_equal(id_area, r_area)
    np.testing.assert_array_equal(hist, r_hist)
    for e in entries:
        S = len(e["segments_info"])
        got, want = ev._entry_tables(e, gt_id, label, G, S), r_entry(e, r_id, label, G, S, K, nll=ev.uncertainty)
        for k in ("pairs", "pred_area", "conf", "cal"):
            np.testing.assert_array_equal(got[k], want[k], err_msg=k)
        assert got["bad"] == want["bad"] == 0
        np.testing.assert_allclose(got["sums"], want["sums"], rtol=1e-6, atol=1e-9)
        if ev.uncertainty:
            rng = np.random.default_rng(S)
            match = np.where(rng.random(S + 1) < 0.5, rng.integers(0, G + 1, S + 1), 0).astype(np.int32)
            match[0] = 0
            (gc, gs), (wc, ws) = ev._vox_tables(e, gt_id, match), r_vox(e, r_id, match)
            np.testing.assert_array_equal(gc, wc)
            np.testing.assert_allclose(gs, ws, rtol=1e-6, atol=1e-9)


@pytest.mark.gpu
@pytest.mark.parametrize("Q", [100, 200, 600])
def test_tables_against_restatement(Q):
    entries = _entries(0, Q=Q)
    sem, ml = _gt(0)
    _compare_tables(MT.Evaluator(len(entries), K, GP.THING_IDS), entries, sem, ml)


@pytest.mark.gpu
def test_calibration_slots_at_fp32_boundaries():
    """Confidences on every fp32 slot boundary, their neighbours, 0 and 1.0: the same slot as torch.bucketize."""
    g = torch.Generator().manual_seed(7)
    size = (32, 32, 8)
    cells = 32 * 32 * 8
    b = BOUNDS
    edges = torch.cat([b, torch.nextafter(b, torch.full_like(b, 2.0)), torch.nextafter(b, torch.full_like(b, -1.0))])
    edges = edges[(edges >= 0) & (edges <= 1)]
    lin = torch.arange(cells)
    conf = edges[torch.randint(0, edges.numel(), (cells,), generator=g)]
    sem = torch.randint(0, K, size, generator=g).to(torch.uint8)
    sem.view(-1)[::13] = 255
    masks = torch.rand((6,) + size, generator=g) < 0.3
    labels = torch.tensor([1, 2, 9, 3, 9, 10])
    S = 5
    probs = torch.softmax(torch.randn(cells, K, generator=g), 1)
    e = {"lin": lin, "panoptic_seg": torch.randint(0, S + 1, (cells,), generator=g).int(),
         "vox_confidence": conf.clone(), "segments_info": [{"id": i + 1, "category_id": 1} for i in range(S)],
         "ssc_lin": lin, "ssc_pred": torch.randint(0, K, (cells,), generator=g).int(), "ssc_confidence": conf,
         "sem_rows": [(probs, torch.arange(cells, dtype=torch.int32))]}
    e = {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in e.items()}
    e["sem_rows"] = [(p.cuda(), c.cuda()) for p, c in e["sem_rows"]]
    ml = {"labels": labels.cuda(), "masks": masks.cuda()}
    ev = MT.Evaluator(1, K, GP.THING_IDS)
    _compare_tables(ev, [e], sem.cuda(), ml)
    t = ev._entry_tables(e, ev._gt_tables(ml["masks"], MT.gt_walk(labels.tolist(), GP.THING_IDS)[0],
                                          sem.cuda().reshape(-1), 5)[0], sem.cuda().reshape(-1), 5, S)
    assert t["cal"][:, 0, 15].sum() > 0 and t["cal"][:, 0, 0].sum() > 0         # 1.0 and 0 / just below 1/15 reached


@pytest.mark.gpu
def test_pasconet_predict_end_to_end():
    """PascoNet.predict(keep_sem_rows=True) on fixture (b)'s scene, evaluated by the device passes, gives the integer
    tables of the restatement fed by ensemble.py's post-processing of the same network outputs."""
    from pasco_b200 import ops
    import make_golden_predict as P_GP
    thr = json.load(open(os.path.join(GOLD, "predict_manifest.json")))["b"]["thresholds"]
    ops.set_precision("fp32")
    net, _ = parity.load_eval(parity.pasconet(2), "m2")
    b = parity.scene(parity.INFER_MANIFEST["cases"]["m2"], 2)
    dev = torch.device("cuda")
    args = (b["in_feats"], b["in_coords"], b["global_min_Cs"], b["global_max_Cs"], b["min_Cs"], b["max_Cs"])
    Ts = P_GP.poses()[:2]
    entries = net.predict(*args, Ts, keep_sem_rows=True, **thr)
    with torch.no_grad():
        ret = net(*args, predict_panop=True, test=True)
    preds = [{"voxel_logits": (p["voxel_logits"].F, p["voxel_logits"].C[:, 1:]), "query_logits": p["query_logits"]}
             for p in ret["panop_predictions"]]
    sems = [(s.F, s.C[:, 1:]) for s in ret["sem_logits_at_scales"][1]]
    ref = _torch_entries(preds, sems, Ts, thr)
    g = torch.Generator().manual_seed(5)
    X, Y, Z = (256, 256, 32)
    sem = torch.randint(0, K, (X, Y, Z), generator=g).to(torch.uint8)
    sem[torch.rand(X, Y, Z, generator=g) < 0.8] = 0
    sem[torch.rand(X, Y, Z, generator=g) < 0.05] = 255
    masks = torch.zeros((len(b["mask_boxes"]), X, Y, Z), dtype=torch.bool)
    for i, (lo, hi) in enumerate(b["mask_boxes"]):
        masks[i, lo[0]:hi[0], lo[1]:hi[1], lo[2]:hi[2]] = True
    ml = {"labels": b["mask_classes"].to(dev), "masks": masks.to(dev)}
    ev, rv = MT.Evaluator(3, K, GP.THING_IDS), RestatedEvaluator(3, K, GP.THING_IDS)
    ev.update(entries, sem.to(dev), ml)
    rv.update(ref, sem.to(dev), ml)
    for got, want in zip(ev.last_scene, rv.last_scene):
        assert {c: f[3:] for c, f in got["pq"].items()} == {c: f[3:] for c, f in want["pq"].items()}
        assert got["pq_pairs"] == want["pq_pairs"] and got["matches"] == want["matches"]
        assert got["completion"] == want["completion"] and got["n_voxels"] == want["n_voxels"]
        for k in ("tps", "fps", "fns"):
            np.testing.assert_array_equal(got[k], want[k])


@pytest.mark.gpu
def test_pair_table_beyond_shared_memory():
    """G = 1500 gt segments x S = 40 predicted ids: 61 k counters take the global-memory path."""
    g = torch.Generator().manual_seed(3)
    size, n, S = (48, 48, 16), 1500, 40
    cells = size[0] * size[1] * size[2]
    sem = torch.randint(0, K, size, generator=g).to(torch.uint8)
    sem.view(-1)[::11] = 255
    masks = torch.rand((n,) + size, generator=g) < 0.01
    labels = torch.tensor([1 + (i % 8) for i in range(n)])
    lin = torch.sort(torch.randperm(cells, generator=g)[:cells // 2])[0]
    pan = torch.randint(0, S + 1, (lin.numel(),), generator=g).to(torch.int32)
    e = {"lin": lin.cuda(), "panoptic_seg": pan.cuda(),
         "segments_info": [{"id": i + 1, "category_id": 1 + i % 8} for i in range(S)],
         "ssc_lin": lin.cuda(), "ssc_pred": torch.randint(0, K, (lin.numel(),), generator=g).to(torch.int32).cuda(),
         "ssc_confidence": torch.rand(lin.numel(), generator=g).cuda()}
    ml = {"labels": labels.cuda(), "masks": masks.cuda()}
    ev = MT.Evaluator(1, K, GP.THING_IDS, uncertainty=False)
    assert (n + 1) * (S + 1) > 200 * 1024 // 4                   # more counters than the shared-memory table holds
    _compare_tables(ev, [e], sem.cuda(), ml)
    ev.update([e], sem.cuda(), ml)
    assert sum(f[3] + f[5] for f in ev.last_scene[0]["pq"].values()) > 0


@pytest.mark.gpu
def test_all_unknown_scene():
    entries = _entries(0)
    sem, ml = _gt(0)
    sem[:] = 255
    ev = MT.Evaluator(len(entries), K, GP.THING_IDS)
    ev.update(entries, sem, ml)
    for d in ev.compute():
        assert d["precision"] == 0 and d["iou"] == 0 and d["count"] == 0
        assert math.isnan(d["empty_ece"]) and math.isnan(d["nonempty_ece"])     # empty partitions: NaN, as upstream
        assert d["mask_ece"] == 0.0 and d["All"]["pq"] == 0


@pytest.mark.gpu
def test_repeat_calls_bit_identical():
    entries = _entries(1)
    sem, ml = _gt(1)
    runs = []
    for _ in range(2):
        ev = MT.Evaluator(len(entries), K, GP.THING_IDS)
        ev.update(entries, sem, ml)
        runs.append((repr(ev.last_scene), repr(ev.compute())))
    assert runs[0] == runs[1]


def _syncs(entries, sem, ml):
    ev = MT.Evaluator(len(entries), K, GP.THING_IDS)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("warn")
    try:
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            ev.update(entries, sem, ml)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    return sum("synchroniz" in str(x.message) for x in w)


@pytest.mark.gpu
def test_syncs_independent_of_q_and_g():
    sem, ml = _gt(0)
    a = _syncs(_entries(0, Q=100), sem, ml)
    b = _syncs(_entries(0, Q=200), sem, ml)
    ml2 = {"labels": torch.cat([ml["labels"], ml["labels"]]), "masks": torch.cat([ml["masks"], ml["masks"]])}
    c = _syncs(_entries(0, Q=100), sem, ml2)
    assert a == b == c and a > 0


@pytest.mark.gpu
def test_input_validation():
    entries = _entries(0)
    sem, ml = _gt(0)
    ev = MT.Evaluator(len(entries), K, GP.THING_IDS)
    with pytest.raises(ValueError, match="masks"):
        ev.update(entries, sem[:128], ml)
    with pytest.raises(ValueError, match="labels"):
        ev.update(entries, sem, {"labels": ml["labels"][:-1], "masks": ml["masks"]})
    with pytest.raises(ValueError, match="n_classes"):
        ev.update(entries, sem, {"labels": ml["labels"] + 30, "masks": ml["masks"]})
    bad = sem.clone()
    bad[0, 0, 0] = 40
    with pytest.raises(ValueError, match="n_classes"):
        ev.update(entries, bad, ml)
    plain = [{k: v for k, v in e.items() if k != "sem_rows"} for e in entries]
    with pytest.raises(ValueError, match="keep_sem_rows"):
        ev.update(plain, sem, ml)
    MT.Evaluator(len(entries), K, GP.THING_IDS, uncertainty=False).update(plain, sem, ml)


@pytest.mark.gpu
def test_rows_outside_the_ground_truth_grid_are_rejected():
    """A label and mask stack that agree with each other but are smaller than the grid the entries were predicted on
    (a 1:2 volume): rejected before anything is accumulated."""
    entries = _entries(0)
    sem, ml = _gt(0)
    ev = MT.Evaluator(len(entries), K, GP.THING_IDS)
    ev.update(entries, sem, ml)
    before = repr(ev.compute())
    small, sml = sem[::2, ::2, ::2].contiguous(), {"labels": ml["labels"], "masks": ml["masks"][:, ::2, ::2, ::2]}
    with pytest.raises(ValueError, match="cell map of 262144 cells"):           # the semantic rows' cell maps
        ev.update(entries, small, sml)
    assert repr(ev.compute()) == before
    plain = MT.Evaluator(len(entries), K, GP.THING_IDS, uncertainty=False)     # the row passes' own bound check
    plain.update(entries, sem, ml)
    before_plain = repr(plain.compute())
    with pytest.raises(ValueError, match="outside the 262144-cell grid"):
        plain.update(entries, small, sml)
    assert repr(plain.compute()) == before_plain
    bad = [dict(e) for e in entries]
    bad[-1]["sem_rows"] = [(p[:, :K - 1].contiguous(), c) for p, c in bad[-1]["sem_rows"]]
    with pytest.raises(ValueError, match="semantic rows"):
        ev.update(bad, sem, ml)
    assert repr(ev.compute()) == before
