"""Evaluation of PascoNet.predict's outputs on the device: the numbers the reference's Net.step_inference(..., eval=True)
reports (net_panoptic_sparse.py:539-765) — PQ†, PQ, SQ, RQ (all / things / stuff, per class), completion precision,
recall and IoU, semantic mIoU, and with `uncertainty` the instance ECE / NLL, voxel ECE and SSC empty / non-empty
ECE / NLL.

    ev = Evaluator(n_entries=M + 1, n_classes=20, thing_ids=THING_IDS, uncertainty=True)
    entries = net.predict(..., keep_sem_rows=True)
    ev.update(entries, semantic_label, mask_label)        # once per scene
    ev.compute()                                          # one dict per entry, the reference's keys
    ev.tables()                                           # the CSV rows of the reference's table printers

Every pass that touches a voxel runs on the kernels of csrc/metrics.cu over the entries' sparse rows: the ground-truth
ids once per scene, then per entry the (gt id, pred id) intersections, the semantic confusion counts with their
calibration bins and NLL, and after matching the voxel calibration bins.  The host finishes small tables: the segment
matching (IoU > 0.5 is unique, no assignment solver), PQStat, ECE from the bins and the pooled instance lists.

Reference behaviour kept on purpose:
  * a gt segment's area is its own mask's sum, counted before unknown zeroing and before later masks overwrite it;
    predicted areas are counted after zeroing; both segment lists keep only ids still present after zeroing;
  * the pair IoU is a float32 division (the reference divides by a torch scalar), and PQStat sums it in float32;
  * the SSC counts skip unknown cells (add_batch's mask); a cell without a semantic row is one-hot class 0;
  * ECE is torchmetrics 1.4's binary_calibration_error(n_bins=15, norm="l1"): 16 slots from
    bucketize(conf, linspace(0, 1, 16), right=True) − 1, so an empty partition gives NaN;
  * SSC and voxel ECE are averaged per scene, NLL is pooled per voxel, instance ECE / NLL are pooled over instances.
The reference's constant placeholders (AUPRC, AUROC, FPR95, ins_brier, mask_nll) and inference_time are not produced.
"""
from __future__ import annotations

from collections import defaultdict
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch
import torch.nn.functional as F

from . import ops
from .predict import THING_IDS

NLL_EPS = 1e-12                     # SSCMetrics.add_batch_ece
INS_NLL_EPS = 1e-8                  # UncertaintyMetrics.get_stats
MATCH_IOU = 0.5                     # the reference's single uncertainty threshold (net_panoptic_sparse.py:198)
VAL_UPDATE_SYNCS = 3                # host synchronisations of Evaluator(uncertainty=False).update for one entry: the mask
                                    # labels (when on the device), the ground-truth counts, the entry's tables


def calibration_error(conf: torch.Tensor, correct: torch.Tensor) -> torch.Tensor:
    """torchmetrics 1.4 binary_calibration_error(conf, correct, n_bins=15, norm="l1"), restated (fp32, as torchmetrics
    computes it): confidences as given, accuracy = the correctness flag, 16 slots, prop = count / count.sum()."""
    conf = conf.reshape(-1).float()
    if not torch.all((conf >= 0) & (conf <= 1)):
        conf = conf.sigmoid()
    acc = correct.reshape(-1).to(conf.dtype)
    bounds = torch.linspace(0, 1, 16, dtype=conf.dtype, device=conf.device)
    idx = torch.bucketize(conf, bounds, right=True) - 1
    count = torch.zeros(16, dtype=conf.dtype, device=conf.device).scatter_add_(0, idx, torch.ones_like(conf))
    conf_bin = torch.nan_to_num(torch.zeros_like(count).scatter_add_(0, idx, conf) / count)
    acc_bin = torch.nan_to_num(torch.zeros_like(count).scatter_add_(0, idx, acc) / count)
    prop = count / count.sum()
    return torch.sum(torch.abs(acc_bin - conf_bin) * prop)


def ece_from_bins(count, sum_conf, sum_correct) -> float:
    """The same ECE from per-slot counts and sums (float64); NaN when every slot is empty."""
    count = np.asarray(count, np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        conf_bin = np.nan_to_num(np.asarray(sum_conf, np.float64) / count)
        acc_bin = np.nan_to_num(np.asarray(sum_correct, np.float64) / count)
        prop = count / count.sum()
    return float(np.sum(np.abs(acc_bin - conf_bin) * prop))


_ONE_SLOT = int(torch.bucketize(torch.tensor([1.0]), ops.CAL_BOUNDS, right=True)[0]) - 1
_NLL_MISS = float(-torch.log(torch.tensor(0.0) + NLL_EPS))      # −log(p + 1e-12) in fp32 at p = 0


class _Cat:
    """PQStatCat: iou sums in float32 once a pair has added to them (the reference's IoU is a float32 tensor)."""
    __slots__ = ("all_iou", "all_n", "iou", "tp", "fp", "fn")

    def __init__(self):
        self.all_iou, self.all_n, self.iou, self.tp, self.fp, self.fn = 0.0, 0.0, 0.0, 0, 0, 0

    def fields(self):
        return (float(self.all_iou), float(self.all_n), float(self.iou), self.tp, self.fp, self.fn)


def _f32(x):
    return np.float32(x)


def pq_average(cats: Dict[int, _Cat], isthing: Optional[bool], thing_ids, ignore_cat_id: int = 0):
    """PQStat.pq_average (panoptic_quality.py:49-93) with its float32 / float64 mix."""
    pq_dagger, pq, sq, rq, n = _f32(0), _f32(0), _f32(0), 0.0, 0
    per_class = {}
    for label, c in cats.items():
        if label == ignore_cat_id:
            continue
        if isthing is not None and isthing != (label in thing_ids):
            continue
        if c.tp + c.fp + c.fn == 0:
            per_class[label] = {"pq": 0.0, "sq": 0.0, "rq": 0.0}
            continue
        n += 1
        den = c.tp + 0.5 * c.fp + 0.5 * c.fn
        pq_c = _f32(c.iou) / _f32(den)
        sq_c = _f32(c.iou) / _f32(c.tp) if c.tp != 0 else _f32(0)
        rq_c = c.tp / den
        per_class[label] = {"pq": float(pq_c), "sq": float(sq_c), "rq": rq_c}
        pq, sq, rq = pq + pq_c, sq + sq_c, rq + rq_c
        if isthing is None:
            pq_dagger = pq_dagger + (pq_c if label in thing_ids else _f32(c.all_iou) / _f32(max(c.all_n, 1)))
    n = max(n, 1)
    return {"pq_dagger": float(pq_dagger / _f32(n)), "pq": float(pq / _f32(n)), "sq": float(sq / _f32(n)),
            "rq": rq / n, "n": n}, per_class


def panoptic_metrics(cats: Dict[int, _Cat], thing_ids) -> Dict:
    """Net.panoptic_metrics (net_panoptic_sparse.py:846-885) without the logging."""
    res = {}
    for name, isthing in (("All", None), ("Things", True), ("Stuff", False)):
        res[name], per_class = pq_average(cats, isthing, thing_ids)
        if name == "All":
            res["per_class"] = per_class
    return res


def gt_walk(labels: Sequence[int], thing_ids):
    """convert_mask_label_to_panoptic_output's walk over the labels (panoptic_quality.py:357-390) without the masks:
    (segment id each mask paints, [(id, category, isthing, index of the mask that created it)])."""
    seg_of, segs, stuff, cur = [], [], {}, 0
    for i, c in enumerate(labels):
        if c == 0:
            seg_of.append(0)
            continue
        isthing = c in thing_ids
        if not isthing and c in stuff:
            seg_of.append(stuff[c])
            continue
        if not isthing:
            stuff[c] = cur + 1
        cur += 1
        seg_of.append(cur)
        segs.append((cur, c, isthing, i))
    return seg_of, segs


def _iou_div(inter: int, union: int):
    return _f32(inter) / _f32(union)


def finish_pq(cats, pairs, pred_area, gt_area, gt_segs, pred_segs, thing_ids, iou_of=_iou_div):
    """pq_compute_single_core (panoptic_quality.py:175-261) and find_matched_segment at threshold 0.5 (:96-164) from
    the device tables.  pairs int [(G+1), (S+1)], pred_area [S+1] after zeroing, gt_area {id: own mask sum};
    gt_segs / pred_segs = [(id, category)] of the segments present after zeroing, in the reference's order.
    Accumulates into cats (a mapping of _Cat that creates a category when first touched, in the reference's order)
    and returns (this scene's per-category fields, PQ matched pairs, uncertainty matches {pred id: gt id}).
    iou_of(intersection, union) gives the float32 IoU of a pair."""
    gcat, pcat = dict(gt_segs), dict(pred_segs)
    scene = defaultdict(_Cat)
    gt_matched, pred_matched, pq_pairs, unc = set(), set(), set(), {}
    g_idx, p_idx = np.nonzero(pairs[1:, 1:])                      # ascending (gt id, pred id), as np.unique orders
    for g, p in zip((g_idx + 1).tolist(), (p_idx + 1).tolist()):
        if g not in gcat or p not in pcat:
            continue
        inter = int(pairs[g, p])
        iou = iou_of(inter, int(pred_area[p]) + int(gt_area[g]) - inter)
        if iou > MATCH_IOU:
            unc[p] = g
        if gcat[g] != pcat[p]:
            continue
        for st in (cats, scene):
            if gcat[g] not in thing_ids:
                st[gcat[g]].all_iou = _f32(st[gcat[g]].all_iou) + iou
                st[gcat[g]].all_n += 1
            if iou > 0.5:
                st[gcat[g]].tp += 1
                st[gcat[g]].iou = _f32(st[gcat[g]].iou) + iou
        if gcat[g] not in thing_ids:
            pred_matched.add(p)
            pq_pairs.add((g, p))
        if iou > 0.5:
            gt_matched.add(g)
            pred_matched.add(p)
            pq_pairs.add((g, p))
    for g, c in gt_segs:
        if g not in gt_matched:
            cats[c].fn += 1
            scene[c].fn += 1
    for p, c in pred_segs:
        if p not in pred_matched:
            cats[c].fp += 1
            scene[c].fp += 1
    return {c: s.fields() for c, s in scene.items()}, sorted(pq_pairs), unc


class _Entry:
    def __init__(self, K):
        self.cats = defaultdict(_Cat)
        self.c_tp = self.c_fp = self.c_fn = 0
        self.tps, self.fps, self.fns = (np.zeros(K, np.int64) for _ in range(3))
        self.empty_ece = self.nonempty_ece = self.ece_count = 0.0
        self.empty_nll = self.nonempty_nll = self.n_empty = self.n_nonempty = 0.0
        self.ins_confs, self.ins_correct, self.ins_probs, self.ins_labels = [], [], [], []
        self.mask_ece = self.count = 0.0


class Evaluator:
    """Accumulates the reference's test metrics over scenes for n_entries predictions per scene (M subnets + the
    ensemble).  uncertainty=False is the reference's `val` mode: PQ and SSC counts only."""

    def __init__(self, n_entries: int, n_classes: int = 20, thing_ids=THING_IDS, uncertainty: bool = True):
        if not 1 <= n_classes <= 64:
            raise ValueError(f"Evaluator: 1 <= n_classes <= 64 (got {n_classes})")
        self.n_entries, self.K, self.uncertainty = int(n_entries), int(n_classes), bool(uncertainty)
        self.thing_ids = tuple(int(t) for t in thing_ids)
        self.reset()

    def reset(self) -> None:
        self._e = [_Entry(self.K) for _ in range(self.n_entries)]
        self.last_scene: List[Dict] = []        # this scene's per-entry tables (PQ fields, matches, SSC counts, ECE)

    # ------------------------------------------------------------------------------------------------
    def _check(self, entries, semantic_label, mask_label):
        """Every input is checked before anything is accumulated: a scene that raises leaves the Evaluator as it was."""
        if len(entries) != self.n_entries:
            raise ValueError(f"Evaluator.update: {len(entries)} entries for {self.n_entries}")
        if not (isinstance(semantic_label, torch.Tensor) and semantic_label.dim() == 3):
            raise ValueError("Evaluator.update: semantic_label must be a tensor [X, Y, Z]")
        dev = semantic_label.device
        masks, labels = mask_label["masks"], mask_label["labels"]
        if not (isinstance(masks, torch.Tensor) and masks.device == dev and masks.dim() == 4
                and tuple(masks.shape[1:]) == tuple(semantic_label.shape)):
            raise ValueError(f"Evaluator.update: masks must be a tensor [n, {', '.join(map(str, semantic_label.shape))}]"
                             f" on {dev}, got {tuple(masks.shape)}")
        labels = [int(v) for v in torch.as_tensor(labels).reshape(-1).tolist()]
        if len(labels) != masks.shape[0]:
            raise ValueError(f"Evaluator.update: {len(labels)} labels for {masks.shape[0]} masks")
        bad = [v for v in labels if not (0 <= v < self.K or v == 255)]
        if bad:
            raise ValueError(f"Evaluator.update: mask class ids {bad} are not below n_classes = {self.K} (or 255)")
        if self.uncertainty and any("sem_rows" not in e for e in entries):
            raise ValueError("Evaluator(uncertainty=True) needs the semantic rows: predict(..., keep_sem_rows=True)")
        for i, e in enumerate(entries):
            groups = [("lin", torch.int64), ("panoptic_seg", torch.int32)], \
                [("ssc_lin", torch.int64), ("ssc_pred", torch.int32), ("ssc_confidence", torch.float32)]
            if self.uncertainty:
                groups[0].append(("vox_confidence", torch.float32))
            for group in groups:
                for k, dt in group:
                    t = e[k]
                    if not (isinstance(t, torch.Tensor) and t.device == dev and t.dtype == dt and t.dim() == 1
                            and t.shape == e[group[0][0]].shape):
                        raise ValueError(f"Evaluator.update: entry {i}: {k} must be {dt} [{e[group[0][0]].shape[0]}] on "
                                         f"{dev}")
        return masks, labels

    def update(self, entries: Sequence[Dict], semantic_label: torch.Tensor, mask_label: Dict) -> None:
        """One scene: entries from predict / postprocess, semantic_label uint8 [X, Y, Z] (255 = unknown), mask_label
        {"labels": [n], "masks": bool [n, X, Y, Z]} — batch["semantic_label_origin"][i], batch["mask_label_origin"][i]
        — on the device.  Raises ValueError on bad input (including entry rows outside the label's grid) and then leaves
        the accumulated metrics untouched."""
        masks, labels = self._check(entries, semantic_label, mask_label)
        K = self.K
        label = semantic_label.to(torch.uint8).contiguous().view(-1)
        seg_of, segs = gt_walk(labels, self.thing_ids)
        G = len(segs)
        gt_id, mask_sum, id_area, hist = self._gt_tables(masks, seg_of, label, G)
        if hist[K]:
            raise ValueError(f"Evaluator.update: {int(hist[K])} semantic labels are not below n_classes = {K} (or 255)")
        tabs = []
        for i, e in enumerate(entries):
            t = self._entry_tables(e, gt_id, label, G, len(e["segments_info"]))
            if t["pred_area"][0] or t["bad"]:
                raise ValueError(f"Evaluator.update: entry {i}: {int(t['pred_area'][0])} rows outside the {label.numel()}"
                                 f"-cell grid or with panoptic ids outside the segments, {t['bad']} semantic rows outside "
                                 f"the grid or predicting outside [0, {K})")
            tabs.append(t)
        gt_area = {sid: int(mask_sum[i]) for sid, _, _, i in segs}
        gt_segs = [(sid, c) for sid, c, _, _ in segs if id_area[sid] > 0]
        self.last_scene = [self._finish(e, acc, t, gt_id, gt_area, gt_segs, hist[:K])
                           for e, acc, t in zip(entries, self._e, tabs)]

    # the counting passes (csrc/metrics.cu); each returns host tables
    def _gt_tables(self, masks, seg_of, label, G):
        """(gt_id on the device, mask sums [n], id areas [G + 1], class histogram [K + 1])."""
        if not label.is_cuda:
            raise ValueError("Evaluator.update: the evaluation passes take CUDA tensors")
        n, cells = masks.shape[0], label.numel()
        m8 = masks.reshape(n, cells).contiguous().view(torch.uint8) if masks.dtype == torch.bool else \
            (masks.reshape(n, cells) != 0).contiguous().view(torch.uint8)
        seg = torch.tensor(seg_of, dtype=torch.int32).pin_memory().to(label.device, non_blocking=True)
        gt_id, counts = ops.eval_gt(m8, seg, label, G, self.K)
        counts = counts.cpu().numpy()
        return gt_id, counts[:n], counts[n:n + G + 1], counts[n + G + 1:]

    def _entry_tables(self, e, gt_id, label, G, S):
        """{pairs [(G+1), (S+1)], pred_area [S+1], conf [K, K] of the known row cells, cal [2, 2, 16], bad, sums [34]}."""
        K = self.K
        t_pairs = (G + 1) * (S + 1) + S + 1
        o_ssc = t_pairs + t_pairs % 2
        o_sum = K * K + 65 + (K * K + 65) % 2
        tab = torch.zeros(o_ssc + o_sum + 68, dtype=torch.int32, device=label.device)
        ops.eval_pairs(e["lin"], e["panoptic_seg"], gt_id, label, G, S, tab[:t_pairs])
        ops.eval_ssc(e["ssc_lin"], e["ssc_pred"], e["ssc_confidence"], label, K,
                     e["sem_rows"] if self.uncertainty else [], tab[o_ssc:])
        host = tab.cpu()
        t = host.numpy()
        return {"pairs": t[:(G + 1) * (S + 1)].reshape(G + 1, S + 1), "pred_area": t[(G + 1) * (S + 1):t_pairs],
                "conf": t[o_ssc:o_ssc + K * K].reshape(K, K).astype(np.int64),
                "cal": t[o_ssc + K * K:o_ssc + K * K + 64].reshape(2, 2, 16).astype(np.int64),
                "bad": int(t[o_ssc + K * K + 64]),
                "sums": host[o_ssc + o_sum:o_ssc + o_sum + 68].view(torch.float64).numpy().reshape(34)}

    def _vox_tables(self, e, gt_id, match):
        """(cal [2, 16] count / correct per slot, confidence sums [16]) for match int32 [S + 1] (pred id → gt id)."""
        dev = gt_id.device
        vt = torch.zeros(64, dtype=torch.int32, device=dev)
        m = torch.from_numpy(match).pin_memory().to(dev, non_blocking=True)
        ops.eval_vox(e["lin"], e["panoptic_seg"], e["vox_confidence"], gt_id, m, vt)
        vh = vt.cpu()
        return vh[:32].numpy().reshape(2, 16), vh[32:].view(torch.float64).numpy()

    # the host finishing of one entry: accumulates into acc, returns the scene's record
    def _finish(self, e, acc: _Entry, t, gt_id, gt_area, gt_segs, hist):
        K = self.K
        S = len(e["segments_info"])
        pairs, pred_area, conf, cal, sums = t["pairs"], t["pred_area"], t["conf"].copy(), t["cal"], t["sums"]

        # panoptic quality and the uncertainty matches
        pred_segs = [(s["id"], s["category_id"]) for s in e["segments_info"] if 0 < s["id"] <= S and pred_area[s["id"]]]
        fields, pq_pairs, unc = finish_pq(acc.cats, pairs, pred_area, gt_area, gt_segs, pred_segs, self.thing_ids)
        rec = {"pq": fields, "pq_pairs": pq_pairs, "matches": sorted((g, p) for p, g in unc.items())}

        # semantic completion over the known cells (add_batch passes y_true != 255 as its mask); a known cell without a
        # row is (class, 0)
        extra = hist.astype(np.int64) - conf.sum(1)
        conf[:, 0] += extra
        tp, fp, fn = int(conf[1:, 1:].sum()), int(conf[0, 1:].sum()), int(conf[1:, 0].sum())
        diag = np.diag(conf)
        acc.c_tp, acc.c_fp, acc.c_fn = acc.c_tp + tp, acc.c_fp + fp, acc.c_fn + fn
        acc.tps += diag
        acc.fps += conf.sum(0) - diag
        acc.fns += conf.sum(1) - diag
        rec.update(completion=(tp, fp, fn), tps=diag.copy(), fps=conf.sum(0) - diag, fns=conf.sum(1) - diag)
        if not self.uncertainty:
            return rec

        # SSC calibration and NLL; the row-less known cells are one-hot class 0: prediction 0, confidence 1.0
        cnt, cor = cal[:, 0].astype(np.float64), cal[:, 1].astype(np.float64)
        csum = sums[:32].reshape(2, 16).copy()
        nll = sums[32:34].copy()
        n_extra = int(extra.sum())
        cnt[0, _ONE_SLOT] += n_extra
        cor[0, _ONE_SLOT] += int(extra[0])
        csum[0, _ONE_SLOT] += n_extra
        nll[0] += (n_extra - int(extra[0])) * _NLL_MISS
        ece = [ece_from_bins(cnt[i], csum[i], cor[i]) for i in range(2)]
        acc.empty_ece += ece[0]
        acc.nonempty_ece += ece[1]
        acc.ece_count += 1
        acc.empty_nll += nll[0]
        acc.nonempty_nll += nll[1]
        acc.n_empty += cnt[0].sum()
        acc.n_nonempty += cnt[1].sum()
        rec.update(empty_ece=ece[0], nonempty_ece=ece[1], nll_sums=(float(nll[0]), float(nll[1])),
                   n_voxels=(float(cnt[0].sum()), float(cnt[1].sum())))

        # instances (compute_ece_panop): an unmatched prediction's NLL target is the dustbin column n_classes
        gcat = dict(gt_segs)
        kept = set(pred_segs)
        segs = [s for s in e["segments_info"] if (s["id"], s["category_id"]) in kept]
        for s in segs:
            g = unc.get(s["id"])
            acc.ins_confs.append(float(s["confidence"]))
            acc.ins_correct.append(g is not None and gcat[g] == s["category_id"])
            acc.ins_labels.append(K if g is None else gcat[g])
        if segs:
            acc.ins_probs.append(torch.stack([s["all_class_probs"] for s in segs]).float())

        # voxel calibration against the matched gt id of every row's segment
        match = np.zeros(S + 1, np.int32)
        for p, g in unc.items():
            match[p] = g
        vc, vs = self._vox_tables(e, gt_id, match)
        mask_ece = ece_from_bins(vc[0], vs, vc[1]) if vc[0].sum() else 0.0
        acc.mask_ece += mask_ece
        acc.count += 1
        rec["mask_ece"] = mask_ece
        return rec

    # ------------------------------------------------------------------------------------------------
    def compute(self) -> List[Dict]:
        """Per entry: SSCMetrics.get_stats, Net.panoptic_metrics and UncertaintyMetrics.get_stats, the reference's keys."""
        out = []
        for a in self._e:
            if a.c_tp != 0:
                p = a.c_tp / (a.c_tp + a.c_fp)
                r = a.c_tp / (a.c_tp + a.c_fn)
                iou = a.c_tp / (a.c_tp + a.c_fp + a.c_fn)
            else:
                p = r = iou = 0
            iou_ssc = a.tps / (a.tps + a.fps + a.fns + 1e-5)
            d = {"precision": p, "recall": r, "iou": iou, "iou_ssc": iou_ssc, "iou_ssc_mean": float(np.mean(iou_ssc[1:]))}
            d.update(panoptic_metrics(a.cats, self.thing_ids))
            if self.uncertainty:
                d["empty_ece"] = a.empty_ece / a.ece_count if a.ece_count else 0
                d["nonempty_ece"] = a.nonempty_ece / a.ece_count if a.ece_count else 0
                d["empty_nll"] = a.empty_nll / a.n_empty if a.n_empty else 0
                d["nonempty_nll"] = a.nonempty_nll / a.n_nonempty if a.n_nonempty else 0
                d["mask_ece"] = a.mask_ece / a.count if a.count else 0
                confs = torch.tensor(a.ins_confs, dtype=torch.float32)
                d["ins_ece"] = float(calibration_error(confs, torch.tensor(a.ins_correct))) if confs.numel() else 0
                if a.ins_probs:
                    probs = torch.cat(a.ins_probs, 0)
                    labels = torch.tensor(a.ins_labels, device=probs.device)
                    d["ins_nll"] = float(F.nll_loss(torch.log(probs + INS_NLL_EPS), labels, reduction="mean"))
                else:
                    d["ins_nll"] = 0.0
                d["count"] = len(a.ins_confs)
            out.append(d)
        return out

    def tables(self, class_names: Optional[Sequence[str]] = None) -> List[str]:
        """The CSV lines of print_metrics_table_panop_ssc, print_metrics_table_panop_per_class and (with uncertainty)
        print_metrics_table_uncertainty (pasco/models/utils.py:22-117); inference time is not measured and prints 0."""
        res = self.compute()
        names = list(class_names) if class_names is not None else [str(c) for c in range(self.K)]
        row = lambda i: "ensemble" if i == len(res) - 1 else f"subnet {i}"          # noqa: E731
        lines = ["=====================================",
                 "method, P, R, IoU, mIoU, All PQ dagger, All PQ, All SQ, All RQ, Thing PQ, Thing SQ, Thing RQ, "
                 "Stuff PQ, Stuff SQ, Stuff RQ"]
        for i, d in enumerate(res):
            v = [d["precision"], d["recall"], d["iou"], d["iou_ssc_mean"], d["All"]["pq_dagger"]] + \
                [d[g][k] for g in ("All", "Things", "Stuff") for k in ("pq", "sq", "rq")]
            lines.append(row(i) + ", " + ", ".join(f"{x * 100:0.2f}" for x in v))
        lines.append("=====================================")
        for metric in ("pq", "sq", "rq"):
            lines += ["==> " + metric, "method, " + ", ".join(names[1:])]
            for i, d in enumerate(res):
                ts = [d["per_class"][c][metric] if c in d["per_class"] else 0 for c in range(1, len(names))]
                lines.append(row(i) + ", " + ", ".join(f"{t * 100:0.2f}" for t in ts))
        if self.uncertainty:
            lines += ["=====================================",
                      "method, ins ece, ins nll, ssc nonempty ece, ssc empty ece, ssc nonempty nll, ssc empty nll,  "
                      "count, inference time"]
            for i, d in enumerate(res):
                lines.append(f"{row(i)},  {d['ins_ece']:0.4f}, {d['ins_nll']:0.4f}, {d['nonempty_ece']:0.4f}, "
                             f"{d['empty_ece']:0.4f}, {d['nonempty_nll']:0.4f}, {d['empty_nll']:0.4f}, {d['count']}, "
                             f"{0.0:0.2f}")
        return lines
