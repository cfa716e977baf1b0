"""The reference's training criterion, term for term (SURVEY.md §8f row 4, "loss path").

`pasco_b200/losses.py` is the compact loss the benchmark closes its fwd+bwd loop with; THIS module restates what
`Net.step` really optimises and is pinned against the reference's own loss code (tests/test_criterion.py ←
tests/golden/make_golden_loss.py, which runs pasco/loss/* from /root/reference and checks its composition against the
reference's real `Net.step`):

  completion_loss     pasco/loss/losses.py:69-179        class-weighted CE (ignore 255) + Lovász-softmax over ALL rows
                                                         inside the scene bounds (a 255 label is background for every
                                                         class there — `ignores=[255]` never matches a class id)
  lovasz_softmax_flat pasco/loss/lovasz.py:186-219       classes "present", optional ignored class ids; all classes in one
                                                         batched sort instead of the per-class Python loop
  HungarianMatcher    pasco/loss/matcher_sparse.py:69-157 cost = 20·focal + 1·(−p_class) + 1·dice over the voxels that carry a
                                                         target and are not unknown, scaled per target by its class
                                                         weight; SciPy assignment on the host exactly where the
                                                         reference has its `C.cpu()`
  SetCriterion        pasco/loss/criterion_sparse.py:56-411  class CE (per-subnet class weights, unreduced → mean over the
                                                         queries), focal + dice on the matched pairs over the known
                                                         voxels, voxel↔query semantic consistency (CE ignore 0 + Lovász
                                                         ignore class 0 on `semantic_inference_v2` logits) — and EVERY aux
                                                         level is matched again (the `indices` argument of the
                                                         reference is never read)
  training_loss       pasco/models/net_panoptic_sparse.py:355-447  the total of `Net.step`: (CE + Lovász)·occ_weight +
                                                         (dice + CE + mask)·panop_weight/M + Σ aux terms/M; the
                                                         main level's ssc terms are computed by the reference but never
                                                         added (the two accumulators stay 0.0) — skipped here

Device-agnostic torch code: a sparse tensor is anything with `.F` [N, C] and `.C` [N, 4] (b, x, y, z) — a
`pasco_b200.me.SparseTensor` on the GPU, a `Rows` tuple in the CPU tests."""
from __future__ import annotations

from typing import Dict, List, NamedTuple, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn.functional as F
from scipy.optimize import linear_sum_assignment

WEIGHTS = {"ssc_ce": 0.3, "ssc_lovasz": 1.0, "loss_ce": 2.0, "loss_mask": 20.0, "loss_dice": 1.0}   # net_panoptic_sparse.py:139-151


class Rows(NamedTuple):
    F: torch.Tensor
    C: torch.Tensor


def lovasz_softmax_flat(logits: torch.Tensor, labels: torch.Tensor, ignores: Sequence[int] = ()) -> torch.Tensor:
    """lovasz.py:186-219 with classes="present": mean over the classes that occur in `labels` and are not in `ignores` of
    the Lovász extension of the Jaccard loss.  One batched sort over [C, P] (no per-class loop, no host round trip)."""
    if logits.shape[0] == 0:
        return logits.sum() * 0.0
    probs = F.softmax(logits, dim=1)
    n_cls = probs.shape[1]
    cls = torch.arange(n_cls, device=labels.device).view(-1, 1)
    fg = (labels.view(1, -1) == cls).to(probs.dtype)                 # [C, P]
    keep = fg.sum(1) > 0
    for c in ignores:
        if 0 <= c < n_cls:
            keep[c] = False
    err = (fg - probs.t()).abs()
    err_sorted, perm = torch.sort(err, dim=1, descending=True)
    fg_sorted = fg.gather(1, perm)
    gts = fg_sorted.sum(1, keepdim=True)
    inter = gts - fg_sorted.cumsum(1)
    union = gts + (1.0 - fg_sorted).cumsum(1)
    jac = 1.0 - inter / union                                        # lovasz_grad, lovasz.py:19-31
    jac = torch.cat([jac[:, :1], jac[:, 1:] - jac[:, :-1]], 1)
    per_class = (err_sorted * jac).sum(1)
    w = keep.to(probs.dtype)
    return (per_class * w).sum() / w.sum().clamp(min=1.0)


def label_weights(class_frequencies, power: float = 1.0 / 3.0) -> torch.Tensor:
    """losses.py:134-140 (SemanticKITTI, power 1/3) / :80-86 (KITTI-360, power 1/1.5)."""
    fr = np.asarray(class_frequencies, dtype=np.float64)
    w = fr / fr.sum()
    return torch.from_numpy(np.power(np.amax(w) / w, power))


def completion_loss(sem_labels: Dict[str, torch.Tensor], sem_logits_at_scales: Dict[int, list], min_Cs, max_Cs,
                    class_frequencies: Dict[str, np.ndarray], power: float = 1.0 / 3.0) -> Tuple[torch.Tensor, torch.Tensor]:
    """losses.py:121-179 → (CE, Lovász), each the mean over every (scale, subnet) pair with at least one row inside the
    subnet's bounds (misc.py:16-27)."""
    ces, lovs = [], []
    for scale, per_subnet in sem_logits_at_scales.items():
        targets = sem_labels[f"1_{scale}"]
        for m in range(len(targets)):
            lg = per_subnet[m]
            dev = lg.F.device
            w = label_weights(class_frequencies[f"1_{scale}"], power).to(device=dev, dtype=lg.F.dtype)
            lo, hi = torch.as_tensor(min_Cs[m]).to(dev).view(1, 3), torch.as_tensor(max_Cs[m]).to(dev).view(1, 3)
            xyz = lg.C[:, 1:]
            inside = ((xyz >= lo) & (xyz <= hi)).all(1)
            if not bool(inside.any()):
                continue
            cell = torch.div(xyz[inside].long() - lo.long(), scale, rounding_mode="floor")
            t = targets[m].to(dev)[cell[:, 0], cell[:, 1], cell[:, 2]].long()
            logits = lg.F[inside]
            ces.append(F.cross_entropy(logits, t, weight=w, ignore_index=255))
            lovs.append(lovasz_softmax_flat(logits, t, ignores=(255,)))
    if not ces:
        return torch.zeros(()), torch.zeros(())
    return torch.stack(ces).mean(), torch.stack(lovs).mean()


def sigmoid_focal(logits: torch.Tensor, targets: torch.Tensor, alpha: float = 0.25, gamma: float = 2.0) -> torch.Tensor:
    """losses.py:45-66, elementwise."""
    p = logits.sigmoid()
    ce = F.binary_cross_entropy_with_logits(logits, targets, reduction="none")
    p_t = p * targets + (1 - p) * (1 - targets)
    return (alpha * targets + (1 - alpha) * (1 - targets)) * ce * (1 - p_t) ** gamma


def dice(logits: torch.Tensor, targets: torch.Tensor) -> torch.Tensor:
    """losses.py:27-42: per column (sums over the voxel dimension 0)."""
    s = logits.sigmoid()
    return 1 - (2 * (s * targets).sum(0) + 1) / (s.sum(0) + targets.sum(0) + 1)


class HungarianMatcher:
    """matcher_sparse.py:69-157.  __call__(query_logits [Q, K+1], mask_logits [N, Q], labels [T], masks [N, T] (0/1),
    class_weight [K+1], unknown [N] bool) → (query idx, target idx), int64 on the host."""

    def __init__(self, cost_class: float = 1.0, cost_mask: float = 20.0, cost_dice: float = 1.0):
        self.cost_class, self.cost_mask, self.cost_dice = cost_class, cost_mask, cost_dice

    @torch.no_grad()
    def cost(self, query_logits, mask_logits, labels, masks, class_weight, unknown) -> torch.Tensor:
        prob = query_logits.softmax(-1)
        ids = labels.long()
        out = mask_logits.t()                                         # [Q, N]
        tgt = masks.t().to(out)                                       # [T, N]
        valid = (tgt.sum(0) > 0) & ~unknown
        out, tgt = out[:, valid], tgt[:, valid]
        cost_class = -prob[:, ids]
        s = out.sigmoid()
        cost_dice = 1 - (2 * s @ tgt.t() + 1) / (s.sum(-1)[:, None] + tgt.sum(-1)[None, :] + 1)
        if out.shape[1] != 0:
            bce_pos = F.binary_cross_entropy_with_logits(out, torch.ones_like(out), reduction="none")
            bce_neg = F.binary_cross_entropy_with_logits(out, torch.zeros_like(out), reduction="none")
            pos = 0.25 * (1 - s) ** 2 * bce_pos
            neg = 0.75 * s ** 2 * bce_neg
            cost_mask = (pos @ tgt.t() + neg @ (1 - tgt).t()) / out.shape[1]
        else:
            cost_mask = torch.zeros_like(cost_dice)
        c = self.cost_mask * cost_mask + self.cost_class * cost_class + self.cost_dice * cost_dice
        return c * class_weight.to(c)[ids][None, :]

    def __call__(self, query_logits, mask_logits, labels, masks, class_weight, unknown):
        c = self.cost(query_logits, mask_logits, labels, masks, class_weight, unknown)
        i, j = linear_sum_assignment(c.float().cpu().numpy())
        return torch.as_tensor(i, dtype=torch.int64), torch.as_tensor(j, dtype=torch.int64)


def semantic_inference(mask_probs: torch.Tensor, query_logits: torch.Tensor) -> Optional[torch.Tensor]:
    """helper.py:7-39 (`semantic_inference_v2`): voxel class logits as the mask-probability-weighted mean of the class logits
    of the queries whose arg-max is not the dustbin; None when every query is dustbin."""
    n_classes = query_logits.shape[-1] - 1
    keep = query_logits.softmax(-1).argmax(-1) != n_classes
    if not bool(keep.any()):
        return None
    p = mask_probs[:, keep] + 1e-8
    return (p / p.sum(1, keepdim=True)) @ query_logits[keep, :-1]


class SetCriterion:
    """criterion_sparse.py:19-411 for one scene per call (the reference's `bs` is 1 per subnet, net_panoptic_sparse.py:417).

    class_weights: one [K+1] tensor per subnet (scripts/train.py:117-123); compl_labelweights [K] (train.py:125-128)."""

    def __init__(self, num_classes: int, class_weights: Sequence[torch.Tensor], compl_labelweights: torch.Tensor,
                 weights: Optional[Dict[str, float]] = None, matcher: Optional[HungarianMatcher] = None):
        self.num_classes = num_classes
        self.class_weights = list(class_weights)
        self.compl_labelweights = compl_labelweights
        self.w = dict(WEIGHTS if weights is None else weights)
        self.matcher = matcher or HungarianMatcher(1.0, self.w["loss_mask"], self.w["loss_dice"])
        # the last __call__'s assignments, one per level (after training_loss or fused_training_loss: the last subnet's);
        # fused_training_loss also leaves every subnet's in subnet_indices
        self.last_indices: List[Tuple[torch.Tensor, torch.Tensor]] = []
        self.subnet_indices: List[List[Tuple[torch.Tensor, torch.Tensor]]] = []

    def level_losses(self, voxel_logits, query_logits, labels, masks_dense, semantic_label, unknown_dense, i_infer: int,
                     min_C, with_ssc: bool = True) -> Dict[str, torch.Tensor]:
        """compute_losses (criterion_sparse.py:239-351) for one output level.  voxel_logits: rows [N, Q] with absolute
        coordinates; query_logits [1, Q, K+1]; masks_dense bool [T, X, Y, Z], semantic_label [X, Y, Z] and unknown_dense
        bool [X, Y, Z] indexed by coordinate − min_C."""
        Fv, dev = voxel_logits.F, voxel_logits.F.device
        cw = self.class_weights[i_infer].to(dev)
        q = query_logits[0]
        cell = voxel_logits.C[:, 1:].long() - torch.as_tensor(min_C).to(dev).long().view(1, 3)
        x, y, z = cell[:, 0], cell[:, 1], cell[:, 2]
        masks = masks_dense.to(dev)[:, x, y, z].t().to(Fv.dtype)       # [N, T]
        unknown = unknown_dense.to(dev)[x, y, z]
        labels = labels.to(dev)
        qi, tj = self.matcher(q, Fv.detach(), labels, masks, cw, unknown)
        self.last_indices.append((qi, tj))
        qi, tj = qi.to(dev), tj.to(dev)
        # loss_labels (:56-81): unreduced weighted CE over the Q queries, then a plain mean
        target_cls = torch.full((q.shape[0],), self.num_classes, dtype=torch.int64, device=dev)
        target_cls[qi] = labels[tj].long()
        loss_ce = (F.cross_entropy(q, target_cls, cw.to(q.dtype), reduction="none") * self.w["loss_ce"]).mean()
        # loss_masks (:83-112): matched pairs over the known voxels, weighted by the class weight of each target
        tw = cw[labels[tj].long()]
        known = ~unknown
        src, tgt = Fv[:, qi][known], masks[:, tj][known]
        loss_mask = ((sigmoid_focal(src, tgt) * tw.unsqueeze(0)).mean(0) * self.w["loss_mask"]).mean()
        loss_dice = (dice(src, tgt) * tw * self.w["loss_dice"]).mean()
        out = {"loss_ce": loss_ce, "loss_mask": loss_mask, "loss_dice": loss_dice}
        if with_ssc:
            out.update(self.ssc_losses(Fv, q, cell, semantic_label))
        return out

    def ssc_losses(self, mask_logits, q, cell, semantic_label) -> Dict[str, torch.Tensor]:
        """compute_ssc_sparse_loss (:182-210), weighted (:337-342)."""
        dev = mask_logits.device
        zero = mask_logits.sum() * 0.0
        logits = semantic_inference(mask_logits.sigmoid(), q)
        if logits is None:
            return {"ssc_ce_loss": zero, "ssc_lovasz_loss": zero}
        t = semantic_label.to(dev)[cell[:, 0], cell[:, 1], cell[:, 2]].long()
        ok = t != 255
        logits, t = logits[ok], t[ok]
        ce = F.cross_entropy(logits, t, weight=self.compl_labelweights.to(logits), ignore_index=0)
        lov = lovasz_softmax_flat(logits, t, ignores=(0,))
        return {"ssc_ce_loss": ce * self.w["ssc_ce"], "ssc_lovasz_loss": lov * self.w["ssc_lovasz"]}

    def __call__(self, pred: Dict, labels, masks_dense, semantic_label, unknown_dense, i_infer: int, min_C,
                 main_ssc: bool = False) -> Dict[str, torch.Tensor]:
        """forward (:353-411): main level + one re-matched pass per aux level (keys `<term>_level<i>`).  main_ssc=False
        skips the main level's ssc terms, which `Net.step` computes and then drops."""
        self.last_indices = []
        losses = self.level_losses(pred["voxel_logits"], pred["query_logits"], labels, masks_dense, semantic_label,
                                   unknown_dense, i_infer, min_C, with_ssc=main_ssc)
        aux = {}
        for i, a in enumerate(pred.get("aux_outputs", [])):
            for k, v in self.level_losses(a["voxel_logits"], a["query_logits"], labels, masks_dense, semantic_label,
                                          unknown_dense, i_infer, min_C).items():
                aux[f"{k}_level{i}"] = v
        losses["loss_aux"] = aux
        return losses


def training_loss(out: Dict, batch: Dict, criterion: SetCriterion, class_frequencies, occ_weight: float = 1.0,
                  panop_weight: float = 1.0, power: float = 1.0 / 3.0):
    """The loss of `Net.step` (net_panoptic_sparse.py:355-447) from a forward output dict (`sem_logits_at_scales`,
    `panop_predictions`) and the reference's batch fields: sem_labels {"1_s": [M, X/s, Y/s, Z/s]}, min_Cs / max_Cs,
    semantic_label [M, X, Y, Z], mask_label [{"labels" [T], "masks" [T, X, Y, Z]}], geo_labels["1_1"] [M, X, Y, Z]
    (255 = unknown).  Returns (total, terms)."""
    ce, lov = completion_loss(batch["sem_labels"], out["sem_logits_at_scales"], batch["min_Cs"], batch["max_Cs"],
                              class_frequencies, power)
    total = (ce + lov) * occ_weight
    terms = {"compl_ce_loss": ce, "compl_lovasz_loss": lov}
    preds = out.get("panop_predictions")
    if not preds:
        return total, terms
    per_subnet = []
    for m, pred in enumerate(preds):
        ml = batch["mask_label"][m]
        unknown = batch["geo_labels"]["1_1"][m] == 255
        per_subnet.append(criterion(pred, ml["labels"], ml["masks"], batch["semantic_label"][m], unknown, m,
                                    batch["min_Cs"][m]))
    return _panoptic_total(total, terms, per_subnet, panop_weight)


def _panoptic_total(total, terms, per_subnet, panop_weight):
    """Net.step's sum of the subnets' criterion outputs (net_panoptic_sparse.py:417-447) onto the completion terms."""
    n = len(per_subnet)
    for ls in per_subnet:
        for k in ("loss_ce", "loss_mask", "loss_dice"):
            terms[k] = terms.get(k, 0.0) + ls[k] / n
        for k, v in ls["loss_aux"].items():
            terms[k] = terms.get(k, 0.0) + v / n
    total = total + (terms["loss_dice"] + terms["loss_ce"] + terms["loss_mask"]) * panop_weight
    for k, v in terms.items():
        if "_level" in k:
            total = total + v
    return total, terms


# ------------------------------------------------------------------------------------------------
# the same objective on the device: grouped setloss kernels (csrc/setloss.cu), one host read per call
# ------------------------------------------------------------------------------------------------
FUSED_SYNCS = 1       # host synchronisations of one fused_training_loss call, whatever M, the levels, N or T
MAX_CLASSES, MAX_KEPT = 64, 128


class DeviceCriterion:
    """The criterion's device driver, shared by `fused_training_loss` (every subnet, level and completion pair of a step)
    and the reference hook's adapters (one level, or one completion-loss call).

    add_pair / add_subnet queue the sampling launches and the counters the host must see; read() launches the kept
    queries and matcher costs of every level, makes the ONE device-to-host copy, decides whether the kernels cover the
    inputs and assigns each level with SciPy; run() launches the matched-pair sums, the semantic-consistency logits and
    every Lovász term, one launch per pass.  Afterwards each pair holds "n_in", "ce" and "lovasz"; each level "qi",
    "tj" (int32, device), "sums" [P, 4], and for a level with ssc "kq", "ssc_logits" (None without a kept query) and
    "ssc_lovasz" (None without a present class other than 0); each subnet "known", "labels", "cw", "lab"."""

    def __init__(self, dev):
        from . import ops
        self.ops, self.dev = ops, dev
        self.parts, self.pairs, self.subnets, self.levels = [], [], [], []

    # ---- queued before the read -------------------------------------------------------------------------------------
    def add_pair(self, sl, target, lo, hi, scale: int, weight):
        """One completion pair (losses.py:121-179): rows `sl` (.F [N, C], .C [N, 4]) against the label volume `target`
        [X, Y, Z] at cell (xyz − lo) // scale for the rows inside [lo, hi]; weight = the CE class weights (host list or
        tensor).  In-bounds rows labelled 255 are background of every class for the Lovász term and ignored by the CE."""
        dev = self.dev
        lo, hi = self.ops.on_device(lo, dev).reshape(1, 3), self.ops.on_device(hi, dev).reshape(1, 3)
        xyz = sl.C[:, 1:]
        inside = ((xyz <= hi) & (xyz >= lo)).all(1)
        cell = (xyz - lo) // scale
        X, Y, Z = target.shape
        ok = inside & (cell >= 0).all(1) & (cell[:, 0] < X) & (cell[:, 1] < Y) & (cell[:, 2] < Z)
        cell = torch.where(ok[:, None], cell, 0).long()
        t = target[cell[:, 0], cell[:, 1], cell[:, 2]].long()
        C_ = sl.F.shape[1]
        cls = torch.where(ok & (t < C_), t, C_)
        counts = torch.zeros(C_ + 1, dtype=torch.int32, device=dev).scatter_add_(
            0, cls, torch.ones_like(cls, dtype=torch.int32))
        stat = torch.cat([torch.stack([inside.sum(), (inside & ~ok).sum()]).to(torch.int32), (counts[:C_] > 0).to(torch.int32)])
        w = weight if torch.is_tensor(weight) else torch.as_tensor(weight, dtype=sl.F.dtype)
        self.pairs.append(dict(F=sl.F, C=C_, w=self.ops.on_device(w, dev).to(sl.F.dtype), t_ce=torch.where(ok, t, 255),
                               t_lov=torch.where(ok, t, -1).to(torch.int32), present=counts[:C_] > 0))
        self.parts.append(("pair", self.pairs[-1], stat))

    def add_subnet(self, C, min_C, masks, unknown, label, labels, class_weight, K: int, levels):
        """One subnet's target sampling (pasco_setloss_sample) and its levels: `levels` a list of (F [N, Q] fp32,
        query_logits [Q, K + 1], with_ssc) whose rows are those of C [N, 4] (b, x, y, z); masks [T, X, Y, Z], unknown
        bool and label [X, Y, Z] at xyz − min_C; labels [T] and class_weight [K + 1] may live on the host."""
        ops, dev = self.ops, self.dev
        T = masks.shape[0]
        bits, flags, lab, stats = ops.setloss_sample(C.to(torch.int32).contiguous(),
                                                     ops.on_device(min_C, dev).reshape(3).to(torch.int32), masks,
                                                     unknown, label, K)
        labels = ops.on_device(labels, dev)
        sub = dict(T=T, K=K, bits=bits, flags=flags, lab=lab, stats=stats, labels=labels, ids=labels.to(torch.int32),
                   cw=ops.on_device(class_weight, dev).float().contiguous())
        # rows of another batch item: left out by the sampling, so not covered
        self.parts.append(("subnet", sub, torch.cat([stats, (C[:, 0] != 0).sum().to(torch.int32).view(1)])))
        self.subnets.append(sub)
        for i, (F_, ql, with_ssc) in enumerate(levels):
            self.levels.append(dict(sub=sub, m=len(self.subnets) - 1, i=i, F=F_, ql=ql.float(), ssc=with_ssc, T=T,
                                    bits=bits, flags=flags, stats=stats, ids=sub["ids"], class_weight=sub["cw"]))

    def add_row_check(self, same: torch.Tensor):
        """A device count that must read 0 for the kernels to cover the call (e.g. rows that differ between levels)."""
        self.parts.append(("check", None, same.to(torch.int32).reshape(1)))

    # ---- the one read -----------------------------------------------------------------------------------------------
    def read(self, matcher, skip_empty: bool = True) -> bool:
        """Launches the kept queries and costs of every level, copies every counter and cost matrix to the host in one
        read and assigns each level.  False: the kernels do not cover the inputs (rows or labels outside the volume,
        rows of another batch item, no labelled row, a completion pair with rows in bounds but no labelled one, more
        than MAX_KEPT kept queries, and — skip_empty False — a pair without a row in bounds)."""
        ops, dev = self.ops, self.dev
        ssc = [lv for lv in self.levels if lv["ssc"]]
        parts = [t for _, _, t in self.parts]
        if self.levels:
            if ssc:
                keep, kept = ops.setloss_keep_group([lv["ql"].detach().contiguous() for lv in ssc])
                for j, lv in enumerate(ssc):
                    lv["keep"] = keep[j]
                parts.append(kept)
            cost = ops.match_cost_group([dict(lv, F=lv["F"].detach().contiguous(),
                                              query_logits=lv["ql"].detach().contiguous()) for lv in self.levels],
                                        matcher.cost_mask, matcher.cost_class, matcher.cost_dice)
            parts = [cost.view(torch.int32)] + parts
        host = torch.cat(parts).cpu()                                                  # the one sync
        at = 0

        def take(k):
            nonlocal at
            at += k
            return host[at - k:at]
        costs = [take(lv["F"].shape[1] * lv["T"]).view(torch.float32).reshape(lv["F"].shape[1], lv["T"])
                 for lv in self.levels]
        ok = True
        for kind, owner, t in self.parts:
            vals = take(t.numel()).tolist()
            if kind == "pair":
                n_in, bad, *present = vals
                owner["n_in"] = n_in
                ok &= not (bad or (n_in and not any(present)) or (n_in == 0 and not skip_empty))
            elif kind == "subnet":
                T = owner["T"]
                present = (vals[T + 2] & 0xFFFFFFFF) | ((vals[T + 3] & 0xFFFFFFFF) << 32)   # unsigned: class 31 unsigned
                owner["known"], owner["present_bits"] = vals[T + 4], present
                ok &= vals[T + 1] == 0 and vals[T + 5] == 0 and present != 0
            else:
                ok &= vals[0] == 0
        if ssc:
            for lv, k in zip(ssc, take(len(ssc)).tolist()):
                lv["kq"] = k
                ok &= k <= MAX_KEPT
        if not ok:
            return False
        import scipy.optimize                 # looked up per call, so that a patched SciPy is the one that assigns
        assigned = [scipy.optimize.linear_sum_assignment(c.numpy()) for c in costs]
        if assigned:
            flat = ops.pinned_to(np.concatenate([np.concatenate([i, j]) for i, j in assigned]).tolist() or [0],
                                 torch.int32, dev)
            at = 0
            for lv, (i, j) in zip(self.levels, assigned):
                P = len(i)
                lv["qi"], lv["tj"], lv["assignment"] = flat[at:at + P], flat[at + P:at + 2 * P], (i, j)
                at += 2 * P
        return True

    # ---- after the read ---------------------------------------------------------------------------------------------
    def run(self):
        ops, dev = self.ops, self.dev
        live = [pr for pr in self.pairs if pr["n_in"] > 0]
        for pr in live:
            pr["ce"] = F.cross_entropy(pr["F"], pr["t_ce"], weight=pr["w"], ignore_index=255)
        lov = [(pr, "lovasz", pr["F"], pr["t_lov"], pr["present"]) for pr in live]
        if self.levels:
            sums = ops.PairSumsGroup.apply([(lv["bits"], lv["T"], lv["flags"], lv["qi"], lv["tj"]) for lv in self.levels],
                                           *[lv["F"] for lv in self.levels])
            at = 0
            for lv in self.levels:
                P = lv["qi"].shape[0]
                lv["sums"], at = sums[at:at + P], at + P
        ssc = [lv for lv in self.levels if lv["ssc"] and lv["kq"] > 0]
        for lv in self.levels:
            lv["ssc_logits"] = lv["ssc_lovasz"] = None
        logits = ops.SscLogitsGroup.apply([(lv["keep"], lv["kq"]) for lv in ssc], *[lv["F"] for lv in ssc],
                                          *[lv["ql"] for lv in ssc]) if ssc else ()
        for lv, lg in zip(ssc, logits):
            sub, K = lv["sub"], lv["sub"]["K"]
            lv["ssc_logits"] = lg
            present = [c != 0 and (sub["present_bits"] >> c) & 1 for c in range(K)]          # ignores=[0]
            if any(present):
                lov.append((lv, "ssc_lovasz", lg, sub["lab"], ops.pinned_to(present, torch.bool, dev)))
        if lov:
            per = ops.LovaszGroup.apply([t[3] for t in lov], *[t[2].float() for t in lov])
            c0 = 0
            for owner, key, x, _, present in lov:
                C_ = x.shape[1]
                w = present.to(per.dtype)
                owner[key] = (per[c0:c0 + C_] * w).sum() / w.sum()
                c0 += C_

    @staticmethod
    def mask_dice(lv, tw):
        """criterion_sparse.py:83-112 from a level's pair sums: per pair (focal over the known rows, dice), each scaled by
        its target's class weight tw [P]."""
        s = lv["sums"]
        return s[:, 0] / lv["sub"]["known"] * tw, (1 - (2 * s[:, 1] + 1) / (s[:, 2] + s[:, 3] + 1)) * tw


def _on_device(v) -> bool:
    """A CUDA tensor, stacked over the subnets or one subnet's, or a list / tuple of per-subnet CUDA tensors (collate_fn
    keeps per-item volumes as lists: each item has its own box)."""
    if isinstance(v, (list, tuple)):
        return len(v) > 0 and all(torch.is_tensor(t) and t.is_cuda for t in v)
    return torch.is_tensor(v) and v.is_cuda


def _covered(out, batch, criterion) -> bool:
    """What can be decided without reading the device: every prediction and label volume is a CUDA tensor, fp32
    logits, at most MAX_CLASSES classes, every level's rows those its subnet samples."""
    sem = out["sem_logits_at_scales"]
    rows = [r for per in sem.values() for r in per]
    preds = out.get("panop_predictions") or []
    if not rows or not all(r.F.is_cuda and r.F.dtype == torch.float32 and 1 <= r.F.shape[1] <= MAX_CLASSES
                           for r in rows):
        return False
    if not all(_on_device(v) for v in batch["sem_labels"].values()):
        return False
    if not preds:
        return True
    vols = [batch["semantic_label"], batch["geo_labels"]["1_1"]] + [ml["masks"] for ml in batch["mask_label"][:len(preds)]]
    if not all(_on_device(v) for v in vols):
        return False
    for p in preds:
        n = p["voxel_logits"].F.shape[0]
        for lv in [p] + list(p.get("aux_outputs", [])):
            F_, ql = lv["voxel_logits"].F, lv["query_logits"]
            if not (F_.is_cuda and F_.dtype == torch.float32 and ql.is_cuda and ql.dtype == torch.float32
                    and ql.shape[-1] - 1 == criterion.num_classes and 1 <= criterion.num_classes <= MAX_CLASSES
                    and ql.shape[-2] == F_.shape[1] <= 4096 and F_.shape[0] == n
                    and lv["voxel_logits"].C.shape == p["voxel_logits"].C.shape):
                return False
    return True


def fused_training_loss(out: Dict, batch: Dict, criterion: SetCriterion, class_frequencies, occ_weight: float = 1.0,
                        panop_weight: float = 1.0, power: float = 1.0 / 3.0):
    """`training_loss` on the grouped setloss kernels (DeviceCriterion): same arguments, same (total, terms) with the
    same keys, every aux level matched again as in the reference.  Target sampling runs once per subnet, every other
    pass once for all levels and subnets; the [Q, T] cost matrices, sampling counters, kept-query counts and each
    completion pair's in-bounds count and present classes reach the host in ONE copy (FUSED_SYNCS), where SciPy assigns
    each level.  Inputs the kernels do not cover — CPU or non-fp32 tensors, more than 64 classes or 128 kept queries,
    no labelled row (in a subnet or in a completion pair with rows in bounds), aux levels on other rows than the main
    level's, and rows or labels outside the volume — run `training_loss` for the whole call.  Afterwards
    criterion.last_indices holds the last subnet's assignments, as after `training_loss`, and criterion.subnet_indices
    every subnet's."""
    if not _covered(out, batch, criterion):
        return training_loss(out, batch, criterion, class_frequencies, occ_weight, panop_weight, power)
    sem_at = out["sem_logits_at_scales"]
    preds = out.get("panop_predictions") or []
    dev = next(iter(sem_at.values()))[0].F.device
    dc = DeviceCriterion(dev)
    for scale, per_subnet in sem_at.items():
        targets = batch["sem_labels"][f"1_{scale}"]
        w = label_weights(class_frequencies[f"1_{scale}"], power).float()
        for m, sl in enumerate(per_subnet[:len(targets)]):
            dc.add_pair(sl, targets[m], batch["min_Cs"][m], batch["max_Cs"][m], scale, w)
    K = criterion.num_classes
    for m, pred in enumerate(preds):
        ml = batch["mask_label"][m]
        lvs = [pred] + list(pred.get("aux_outputs", []))
        C0 = pred["voxel_logits"].C
        dc.add_subnet(C0, batch["min_Cs"][m], ml["masks"], batch["geo_labels"]["1_1"][m] == 255,
                      batch["semantic_label"][m], ml["labels"], criterion.class_weights[m], K,
                      [(lv["voxel_logits"].F, lv["query_logits"][0], i > 0) for i, lv in enumerate(lvs)])
        for lv in lvs[1:]:
            C = lv["voxel_logits"].C
            if C is not C0:
                dc.add_row_check((C != C0).any(1).sum())
    if not dc.read(criterion.matcher):
        return training_loss(out, batch, criterion, class_frequencies, occ_weight, panop_weight, power)
    dc.run()

    live = [pr for pr in dc.pairs if pr["n_in"] > 0]
    if live:
        ce, lov = torch.stack([pr["ce"] for pr in live]).mean(), torch.stack([pr["lovasz"] for pr in live]).mean()
    else:
        ce, lov = torch.zeros((), device=dev), torch.zeros((), device=dev)
    total = (ce + lov) * occ_weight
    terms = {"compl_ce_loss": ce, "compl_lovasz_loss": lov}
    criterion.subnet_indices = [[tuple(torch.as_tensor(a, dtype=torch.int64) for a in lv["assignment"])
                                 for lv in dc.levels if lv["m"] == m] for m in range(len(preds))]
    if criterion.subnet_indices:
        criterion.last_indices = criterion.subnet_indices[-1]
    if not preds:
        return total, terms

    wd = criterion.w
    per_subnet = []
    for m, sub in enumerate(dc.subnets):
        ls, aux = None, {}
        for lv in [lv for lv in dc.levels if lv["m"] == m]:
            q, cw = lv["ql"], sub["cw"]
            qi, tj = lv["qi"].long(), lv["tj"].long()
            target_cls = torch.full((q.shape[0],), K, dtype=torch.int64, device=dev)
            target_cls[qi] = sub["labels"][tj].long()
            d = {"loss_ce": (F.cross_entropy(q, target_cls, cw.to(q.dtype), reduction="none") * wd["loss_ce"]).mean()}
            loss_mask, loss_dice = DeviceCriterion.mask_dice(lv, cw[sub["labels"][tj].long()])
            d["loss_mask"] = (loss_mask * wd["loss_mask"]).mean()
            d["loss_dice"] = (loss_dice * wd["loss_dice"]).mean()
            if lv["ssc"]:
                zero = lv["F"].sum() * 0.0
                if lv["ssc_logits"] is not None:
                    t = torch.where(sub["lab"] < 0, 0, sub["lab"]).long()
                    d["ssc_ce_loss"] = F.cross_entropy(lv["ssc_logits"], t, weight=dc.ops.on_device(
                        criterion.compl_labelweights, dev).float(), ignore_index=0) * wd["ssc_ce"]
                    lv_lov = lv["ssc_lovasz"] if lv["ssc_lovasz"] is not None else lv["ssc_logits"].sum() * 0.0
                    d["ssc_lovasz_loss"] = lv_lov * wd["ssc_lovasz"]
                else:
                    d["ssc_ce_loss"], d["ssc_lovasz_loss"] = zero, zero
                for k, v in d.items():
                    aux[f"{k}_level{lv['i'] - 1}"] = v
            else:
                ls = d
        ls["loss_aux"] = aux
        per_subnet.append(ls)
    return _panoptic_total(total, terms, per_subnet, panop_weight)
