"""Panoptic scene completion with uncertainty: PascoNet.predict, the engine's form of what scripts/eval.py gets from the
reference's Net.forward(..., Ts, return_ensemble=True) (net_panoptic_sparse.py:210-310) followed by Net.step_inference's
panoptic_inference on every subnet and on the ensemble (net_panoptic_sparse.py:539-648, helper.py:91-303).

Everything after the forward runs on the kernels of csrc/panoptic.cu, on sparse rows of the 256x256x32 reference grid:

  warp            every reference cell looks up the nearest source voxel under the subnet's pose (pasco_pose_lookup), the
                  row compaction turns the cell map into ascending cells `lin` (ME.to_sparse order) and source rows
  activate        sigmoid (masks, with bf16 planes and column sums for the IoU) or softmax (semantic logits) of those rows
  semantic        mean of the M class distributions per cell (an absent subnet counts as one-hot class 0)
  masks           subnet 0 is the anchor; every later subnet is matched to it by soft IoU (a K = 1 weight gradient, then
                  SciPy's linear_sum_assignment on the host, as in the reference) and averaged into it on the union rows
  panoptic        pass 1 (winner record per voxel, integer areas per query), the sequential segment walk on one device
                  thread, pass 2 (labels and confidences); the segment records are the one copy to the host per entry

The torch restatement in ensemble.py is the reference these kernels are tested against.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import numpy as np
import torch
import torch.nn.functional as F

from . import ops

SCENE = (256, 256, 32)
THING_IDS = (1, 2, 3, 4, 5, 6, 7, 8)          # pasco/data/semantic_kitti/params.py


def _coords4(c: torch.Tensor) -> torch.Tensor:
    """[N, 4] (batch, x, y, z) or [N, 3] rows → int32 [N, 4] with batch index 0."""
    c = c[:, -3:].to(torch.int32)
    return torch.cat([torch.zeros_like(c[:, :1]), c], 1).contiguous()


def warp(coords: torch.Tensor, T: torch.Tensor, size=SCENE):
    """Rows of a subnet (integer coords in its augmented frame) → (lin int32 [N'] ascending reference cells,
    cell_row int32 [cells] = row index at each cell or −1, src int32 [N'] = the source row of every new row)."""
    table, _ = ops.hash_insert(_coords4(coords))
    cell_src, mask = ops.pose_lookup(table, T, size)
    lin, cell_row, _ = ops.compact(mask)
    return lin, cell_row, ops.lookup_rows(cell_src, lin)


def _drop_zero_rows(prob: torch.Tensor, lin: torch.Tensor, nz: torch.Tensor):
    """ME.to_sparse drops rows whose mask probabilities are all zero."""
    kept, _, n = ops.compact(nz)
    if n == prob.shape[0]:
        return prob, lin
    return ops._gather_rows(prob, kept), ops.lookup_rows(lin, kept)


def _segments(records: torch.Tensor, query_probs: torch.Tensor) -> List[Dict]:
    r = records.numpy()
    out = []
    for s in range(int(r[0])):
        q, cls, conf, thing = r[1 + 4 * s: 5 + 4 * s]
        out.append({"id": s + 1, "isthing": bool(thing), "category_id": int(cls), "query_id": int(q),
                    "confidence": float(np.array(conf, dtype=np.int32).view(np.float32)),
                    "all_class_probs": query_probs[int(q)]})
    return out


def postprocess(preds: Sequence[Dict], sems: Sequence, Ts: Sequence[torch.Tensor], *, thing_ids=THING_IDS,
                overlap_threshold: float = 0.4, object_mask_threshold: float = 0.7, iou_threshold: float = 0.2,
                size=SCENE, matches: Optional[list] = None, keep_sem_rows: bool = False) -> List[Dict]:
    """preds[m] = {"voxel_logits": (logits [N_m, Q], coords [N_m, 3 or 4]), "query_logits": [1, Q, K1]} and sems[m] =
    (semantic logits [S_m, K], coords) of subnet m, in the subnet's frame under pose Ts[m].  Returns M + 1 entries (the
    subnets, then the ensemble); `matches` (a list) receives the (anchor, subnet) Hungarian assignment of every step.
    keep_sem_rows: every entry also holds "sem_rows", the (softmax rows [n, K], cell map int32 [cells]) pairs its
    semantic output averaged — the subnet's own pair, all M for the ensemble — so that p[c] of the class distribution
    can be evaluated at any cell (metrics.Evaluator's NLL)."""
    M = len(preds)
    if not 1 <= M <= 8:
        raise ValueError(f"predict: 1 to 8 subnets (the semantic ensemble kernel's limit), got {M}")
    sem_rows = semantic_rows(sems, Ts, size)
    ssc, gate = semantic(sem_rows, size)
    rows, qprobs = mask_rows(*mask_warps(preds, Ts, size), gate, iou_threshold=iou_threshold, size=size, matches=matches)
    entries = []
    for (prob, lin), qp, (s_lin, s_pred, s_conf) in zip(rows, qprobs, ssc):
        pan, sem, conf, records = ops.panoptic(prob, qp[0], overlap_threshold, object_mask_threshold, thing_ids)
        entries.append({"lin": lin.long(), "panoptic_seg": pan, "semantic_seg": sem, "vox_confidence": conf,
                        "segments_info": _segments(records, qp[0]), "ssc_lin": s_lin.long(), "ssc_pred": s_pred,
                        "ssc_confidence": s_conf, "query_probs": qp[0]})
    if keep_sem_rows:
        for m, e in enumerate(entries):
            e["sem_rows"] = [(p, cell) for p, _, cell in (sem_rows[m:m + 1] if m < M else sem_rows)]
    return entries


def semantic_rows(sems: Sequence, Ts: Sequence[torch.Tensor], size=SCENE) -> List[tuple]:
    """The semantic logits of every subnet warped to the reference grid: [(softmax rows fp32 [n, K], lin int32 [n]
    ascending cells, cell map int32 [cells])]."""
    out = []
    for (s_logits, s_coords), T in zip(sems, Ts):
        s_lin, s_cell, s_src = warp(s_coords, T, size)
        out.append((ops.softmax_rows(s_logits, s_src), s_lin, s_cell))
    return out


def semantic(sem_rows: Sequence[tuple], size=SCENE):
    """Semantic completion (ensembler.py:160-187): every subnet on its own rows, the ensemble on the union of the rows →
    ([(lin, argmax int32, max fp32)] for the M subnets and the ensemble, the ensemble's occupancy gate uint8 [cells])."""
    cells = int(size[0]) * int(size[1]) * int(size[2])
    dev = sem_rows[0][0].device
    ssc = [(lin,) + ops.sem_ensemble([p], [cell], lin) for p, lin, cell in sem_rows]
    union = torch.zeros(cells, dtype=torch.uint8, device=dev)
    for _, _, cell in sem_rows:
        ops.cell_mask_or(cell, union)
    u_lin, _, _ = ops.compact(union)
    gate = torch.zeros(cells, dtype=torch.uint8, device=dev)
    ssc.append((u_lin,) + ops.sem_ensemble([p for p, _, _ in sem_rows], [c for _, _, c in sem_rows], u_lin, gate))
    return ssc, gate


def mask_warps(preds: Sequence[Dict], Ts: Sequence[torch.Tensor], size=SCENE):
    """The sigmoid rows of every subnet on the reference grid (ensembler.py:36-64) → (per subnet: dict of the
    probabilities, cells, cell map, bf16 planes and column sums when M > 1, non-zero row flags; the M query class
    probabilities [1, Q, K1])."""
    M = len(preds)
    masks, qprobs = [], []
    for m in range(M):
        logits, coords = preds[m]["voxel_logits"]
        lin, cell_row, src = warp(coords, Ts[m], size)
        prob, planes, colsum, nz = ops.mask_rows_sigmoid(logits, src, planes=M > 1)
        masks.append(dict(prob=prob, lin=lin, cell=cell_row, planes=planes, colsum=colsum, nz=nz))
        qprobs.append(F.softmax(preds[m]["query_logits"].detach().float(), -1))
    return masks, qprobs


def mask_rows(masks: Sequence[Dict], qprobs: Sequence[torch.Tensor], gate: torch.Tensor, *, iou_threshold: float = 0.2,
              size=SCENE, matches: Optional[list] = None):
    """The mask ensemble (ensembler.py:66-113) on mask_warps' rows: the running average of the matched queries on the
    union rows, with the mean-IoU keep and the occupancy gate.  Returns M + 1 (probabilities fp32 [n, q], lin int32 [n]
    ascending cells) with all-zero rows dropped (ME.to_sparse), and the M + 1 query class probabilities [1, q, K1]."""
    from scipy.optimize import linear_sum_assignment
    M = len(masks)
    dev = masks[0]["prob"].device
    cells = int(size[0]) * int(size[1]) * int(size[2])
    Q = masks[0]["prob"].shape[1]
    qprobs = list(qprobs)

    # running average of the matched queries on the union rows
    a = masks[0]
    a_q = qprobs[0].clone()
    ious = []
    cols = torch.arange(Q, dtype=torch.int32, device=dev)
    if M == 1:
        ens = ops.mask_merge(a["prob"], a["cell"], None, None, a["lin"], cols, None, 0, gate, planes=False)
        ens_prob, ens_lin = _drop_zero_rows(ens[0], a["lin"], ens[3])
    for i in range(1, M):
        b = masks[i]
        gated = ops.soft_iou(a["prob"], a["planes"], a["colsum"], b["prob"], b["planes"], b["colsum"],
                             ops.lookup_rows(a["cell"], b["lin"]), iou_threshold).cpu().numpy()
        ai, bi = linear_sum_assignment(1.0 - gated)                                    # the reference's host crossing
        if matches is not None:
            matches.append((ai, bi))
        ious.append(torch.from_numpy(gated[ai, bi]))
        ai_t, bi_t = torch.as_tensor(ai, device=dev), torch.as_tensor(bi, device=dev)
        a_q[:, ai_t] = (a_q[:, ai_t] * i + qprobs[i][:, bi_t]) / (i + 1)
        b_of = np.full(Q, -1, dtype=np.int32)
        b_of[ai] = bi
        union = torch.zeros(cells, dtype=torch.uint8, device=dev)
        ops.cell_mask_or(a["cell"], union)
        ops.cell_mask_or(b["cell"], union)
        lin, cell, _ = ops.compact(union)
        if i < M - 1:
            prob, planes, colsum, nz = ops.mask_merge(a["prob"], a["cell"], b["prob"], b["cell"], lin, cols,
                                                      torch.as_tensor(b_of, device=dev), i)
            a = dict(prob=prob, lin=lin, cell=cell, planes=planes, colsum=colsum)
            continue
        # last step: the mean-IoU keep, the ensembled occupancy gate and the all-zero-row drop in the same pass
        keep = (torch.stack(ious, 0).mean(0) > iou_threshold).numpy()
        kept = np.nonzero(keep)[0].astype(np.int32)
        if len(kept) == 0:                       # no query kept: every row is all zeros and ME.to_sparse drops it
            ens_prob, ens_lin = torch.zeros(0, 0, device=dev), lin[:0]
        else:
            prob, _, _, nz = ops.mask_merge(a["prob"], a["cell"], b["prob"], b["cell"], lin,
                                            torch.as_tensor(kept, device=dev), torch.as_tensor(b_of[kept], device=dev), i,
                                            gate, planes=False)
            ens_prob, ens_lin = _drop_zero_rows(prob, lin, nz)
        a_q = a_q[:, torch.as_tensor(keep, device=dev)]
    rows = [_drop_zero_rows(mk["prob"], mk["lin"], mk["nz"]) for mk in masks] + [(ens_prob, ens_lin)]
    return rows, qprobs + [a_q]


# ------------------------------------------------------------------------------------------------
# Net.step's per-step evaluation (net_panoptic_sparse.py:425-475): one subnet of a training forward, in its own box
# ------------------------------------------------------------------------------------------------
STEP_ENTRY_SYNCS = 2    # host synchronisations per subnet of step_entries: the box check, then the segment records
                        # (one more per call reads min_Cs / max_Cs when they are device tensors)


def step_box(min_C, max_C):
    """(min_C, max_C, size) as host int tuples: size = compute_scene_size(min_C, max_C, scale=8) (misc.py:30), the box
    of ceil((max − min + 1) / 8)·8 cells per axis from min_C that Net.step evaluates a subnet in."""
    lo, hi = (torch.as_tensor(v).reshape(-1)[-3:] for v in (min_C, max_C))
    dev = lo.device if lo.is_cuda else hi.device
    both = torch.cat([lo.to(dev, torch.int64), hi.to(dev, torch.int64)]).cpu().tolist()
    lo, hi = both[:3], both[3:]
    size = tuple(int(np.ceil((h - l + 1) / 8.0)) * 8 for l, h in zip(lo, hi))
    if min(size) <= 0:
        raise ValueError(f"step_entries: empty box from min_C {lo} to max_C {hi}")
    return tuple(lo), tuple(hi), size


def _outside_rows_host(C: torch.Tensor, lo, size) -> int:
    xyz = C[:, -3:].long() - torch.tensor(lo).view(1, 3)
    return int(((xyz < 0) | (xyz >= torch.tensor(size).view(1, 3))).any(1).sum())


def step_entries(out: Dict, batch: Dict, subnets: Sequence[int], *, thing_ids=THING_IDS, overlap_threshold: float = 0.4,
                 object_mask_threshold: float = 0.7) -> List[Dict]:
    """One entry per listed subnet i of a training-mode forward output `out` (PascoNet.forward(..., predict_panop=True)),
    in the format postprocess emits, for metrics.Evaluator(n_entries=1, uncertainty=False): what Net.step evaluates
    every training step (net_panoptic_sparse.py:430-459), on rows instead of dense volumes.

    The box is min_C = batch["min_Cs"][i] with step_box's size; `lin` and `ssc_lin` are cells (coord − min_C) of it,
    ascending.  The masks are the sigmoid of panop_predictions[i]["voxel_logits"] with the softmax of its query logits
    through the panoptic passes; every mask row must lie in the box (PascoNet.predict_panop crops to it), a row outside
    raises.  The semantics are the softmax of the scale-1 sem_logits_at_scales[1][i] rows inside [min_C, max_C]
    (prune_outside_coords; other rows are dropped): ssc_pred the argmax, ssc_confidence the max.  The reference densifies zero logits at the box
    cells without a row, whose softmax is uniform with argmax class 0; Evaluator counts a known cell without a row as
    prediction 0, so its SSC counts are the reference's without those cells being written.  batch["semantic_label"][i]
    must have the box's shape.  ValueError on bad subnet indices, a label of another shape, rows outside the box or
    two rows at one cell, and CPU tensors.  STEP_ENTRY_SYNCS host synchronisations per subnet, whatever Q."""
    preds = out.get("panop_predictions") or []
    subnets = list(subnets)
    bad = [i for i in subnets if not (isinstance(i, (int, np.integer)) and not isinstance(i, bool) and 0 <= i < len(preds))]
    if bad:
        raise ValueError(f"step_entries: subnets {bad} are not indices of the {len(preds)} panoptic predictions")
    entries = []
    for i in subnets:
        i = int(i)
        lo, hi, size = step_box(batch["min_Cs"][i], batch["max_Cs"][i])
        label = batch["semantic_label"][i]
        if tuple(label.shape) != size:
            raise ValueError(f"step_entries: subnet {i}: semantic_label has shape {tuple(label.shape)}, the box from "
                             f"{list(lo)} is {list(size)}")
        vl, ql, sl = preds[i]["voxel_logits"], preds[i]["query_logits"], out["sem_logits_at_scales"][1][i]
        if not all(t.is_cuda for t in (vl.F, vl.C, ql, sl.F, sl.C)):
            n = _outside_rows_host(vl.C, lo, size)
            if n:
                raise ValueError(f"step_entries: subnet {i}: {n} mask rows outside the box {list(size)} at {list(lo)}")
            raise ValueError("step_entries: the panoptic and semantic passes take CUDA tensors")
        entries.append(_step_entry(i, vl, ql, sl, lo, hi, size, thing_ids, overlap_threshold, object_mask_threshold))
    return entries


def _step_entry(i, vl, ql, sl, lo, hi, size, thing_ids, overlap_threshold, object_mask_threshold) -> Dict:
    counts = torch.zeros(4, dtype=torch.int32, device=vl.F.device)
    m_cell, m_mask = ops.box_cells(vl.C, lo, [l + s - 1 for l, s in zip(lo, size)], size, counts[:2])   # the whole box
    s_cell, s_mask = ops.box_cells(sl.C, lo, hi, size, counts[2:])                        # prune_outside_coords' bounds
    m_out, m_dup, s_out, s_dup = counts.cpu().tolist()                                     # the box check
    if m_out or m_dup or s_dup:
        raise ValueError(f"step_entries: subnet {i}: {m_out} mask rows outside the box {list(size)} at {list(lo)}; "
                         f"{m_dup} mask rows and {s_dup} semantic rows at a cell another row holds")
    lin, _, _ = ops.compact(m_mask, total=vl.F.shape[0])
    prob = ops.mask_rows_sigmoid(vl.F, ops.lookup_rows(m_cell, lin), planes=False)[0]
    qp = F.softmax(ql.detach().float(), -1)[0]
    pan, sem, conf, records = ops.panoptic(prob, qp, overlap_threshold, object_mask_threshold, thing_ids)   # records
    s_lin, s_new, _ = ops.compact(s_mask, total=sl.F.shape[0] - s_out)           # s_new: cell → row of s_lin's order
    s_pred, s_conf = ops.sem_ensemble([ops.softmax_rows(sl.F, ops.lookup_rows(s_cell, s_lin))], [s_new], s_lin)
    return {"lin": lin.long(), "panoptic_seg": pan, "semantic_seg": sem, "vox_confidence": conf,
            "segments_info": _segments(records, qp), "ssc_lin": s_lin.long(), "ssc_pred": s_pred,
            "ssc_confidence": s_conf, "query_probs": qp}


def evaluate_step(out: Dict, batch: Dict, metrics: Dict, *, thing_ids=THING_IDS, overlap_threshold: float = 0.4,
                  object_mask_threshold: float = 0.7) -> None:
    """Net.step's evaluate_all(compute_uncertainty=False) calls (net_panoptic_sparse.py:425-475): metrics = {subnet:
    metrics.Evaluator(n_entries=1, uncertainty=False)} accumulates step_entries' entry of that subnet against
    batch["semantic_label"][i] and batch["mask_label"][i] — pq_stat["train"][i] and ssc_metrics["train"][i].  Every
    entry is built before any Evaluator is touched."""
    subnets = sorted(metrics)
    with torch.no_grad():
        entries = step_entries(out, batch, subnets, thing_ids=thing_ids, overlap_threshold=overlap_threshold,
                               object_mask_threshold=object_mask_threshold)
        for i, e in zip(subnets, entries):
            metrics[i].update([e], batch["semantic_label"][i], batch["mask_label"][i])


_DENSE = {"panoptic_seg": ("lin", 0.0), "semantic_seg": ("lin", 0.0), "vox_confidence": ("lin", 0.0),
          "ssc_pred": ("ssc_lin", 0.0), "ssc_confidence": ("ssc_lin", 1.0)}


def to_dense(entry: Dict, key: str, size=SCENE) -> torch.Tensor:
    """The reference's dense [X, Y, Z] volume of one per-row output of an entry (metric code indexes these).  Cells
    without a row hold the reference's fill: 1.0 for ssc_confidence (an empty cell is one-hot class 0), 0 elsewhere."""
    rows_key, fill = _DENSE[key]
    lin, v = entry[rows_key], entry[key]
    X, Y, Z = (int(s) for s in size)
    coords = torch.stack([torch.zeros_like(lin), lin // (Y * Z), (lin // Z) % Y, lin % Z], 1).to(torch.int32).contiguous()
    dense = torch.full((1, 1, X, Y, Z), fill, dtype=torch.float32, device=v.device)
    mc, st = ops._geom((0, 0, 0), (1, 1, 1))
    ops.call("pasco_to_dense", ops.ptr(v.float().view(-1, 1).contiguous()), ops.ptr(coords), lin.shape[0], 1, mc, st,
             ops.ptr(dense), 1, X, Y, Z, None)
    dense = dense.view(X, Y, Z)
    return dense.to(v.dtype) if v.dtype != torch.float32 else dense


def predict(net, in_feats, in_coords, global_min, global_max, min_Cs, max_Cs, Ts=None, *, thing_ids=THING_IDS,
            overlap_threshold=0.4, object_mask_threshold=0.7, iou_threshold=0.2, scene_size=SCENE,
            keep_sem_rows: bool = False) -> List[Dict]:
    """PascoNet.predict: the eval forward (forward(test=True), no gradients), then postprocess."""
    if net.training:
        raise RuntimeError("PascoNet.predict runs the eval forward: call net.eval() first")
    M = net.n_infers
    if Ts is None:
        Ts = [torch.eye(4) for _ in range(M)]
    if len(Ts) != M:
        raise ValueError(f"PascoNet.predict: {len(Ts)} poses for {M} subnets")
    with torch.no_grad():
        ret = net(in_feats, in_coords, global_min, global_max, min_Cs, max_Cs, predict_panop=True, test=True)
        preds = [{"voxel_logits": (p["voxel_logits"].F, p["voxel_logits"].C), "query_logits": p["query_logits"]}
                 for p in ret["panop_predictions"]]
        sems = [(s.F, s.C) for s in ret["sem_logits_at_scales"][1]]
        return postprocess(preds, sems, Ts, thing_ids=thing_ids, overlap_threshold=overlap_threshold,
                           object_mask_threshold=object_mask_threshold, iou_threshold=iou_threshold, size=scene_size,
                           keep_sem_rows=keep_sem_rows)
