"""Golden vectors for predict.step_entries + metrics.Evaluator — BUILD CONTAINER ONLY: runs the reference's OWN code of
Net.step's per-step evaluation (net_panoptic_sparse.py:425-475) from the upstream checkout on the CPU (MinkowskiEngine =
the oracle shim), over a synthetic M = 2 training output:

  * panoptic_inference (helper.py:91-303) on the sigmoid of each subnet's voxel logits and the softmax of its query
    logits, with min_C, scene_size = compute_scene_size(min_C, max_C, scale=8) and input_query_logit=False;
  * prune_outside_coords (misc.py:16-27) of the scale-1 semantic logits, .dense over the box from min_C, softmax and
    its max;
  * Net.evaluate_all(compute_uncertainty=False) (net_panoptic_sparse.py:650-695), called unbound on a stub carrying
    thing_ids and n_classes, into one PQStat and one SSCMetrics per subnet, accumulated over two steps.

    python tests/golden/make_golden_step_eval.py

The output covers a non-zero min_C whose box (32 x 24 x 16) is larger than [min_C, max_C], mask rows on the box's faces
(also past max_C), semantic rows outside [min_C, max_C] (pruned), labelled box cells without a semantic row, 255 labels,
a subnet with no kept query (subnet 1 of step 0), thing and stuff segments with two queries of one stuff class merged,
and two accumulated steps.

Stored (step_eval_m2.npz): the inputs (per step s and subnet m: vox_C / vox_F / query / sem_C / sem_F, the labels and
masks, min_C / max_C) and, after each step, per subnet: the PQStat per-category fields (all_iou, all_n, iou, tp, fp, fn)
and the SSC completion tp / fp / fn and per-class tps / fps / fns.  To keep the file small the voxel and semantic logits
are multiples of 1/16 in [-127/16, 127/16], stored as int8 counts of 1/16 (exact in fp32), and the coordinates as int8;
the reference runs on exactly those values.
"""
import os
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))

import numpy as np  # noqa: E402
import torch  # noqa: E402

K, K1, Q, M, STEPS = 20, 21, 12, 2, 2
MIN_C, MAX_C = (8, -4, 0), (35, 15, 11)          # box = compute_scene_size → (32, 24, 16), past max_C on every axis
THING_IDS = [1, 2, 3, 4, 5, 6, 7, 8]
OVERLAP, OBJECT_MASK = 0.4, 0.7
LOGIT_UNIT = 16                                    # logits are integers / LOGIT_UNIT, stored as int8
INT8_KEYS = ("vox_C", "vox_F", "sem_C", "sem_F")


def quantise(x):
    return torch.round(x * LOGIT_UNIT).clamp(-127, 127) / LOGIT_UNIT


def to_stored(k, v):
    """The .npz form of one synthetic() tensor (the test's _case undoes it)."""
    if k in ("vox_F", "sem_F"):
        return (v * LOGIT_UNIT).round().to(torch.int8).numpy()
    if k in ("vox_C", "sem_C"):
        return v.to(torch.int8).numpy()
    return v.numpy()
# per query: (class, box lo, box hi) in box cells; class 0 / K1 - 1 = not kept, two queries of stuff class 9 merge
OBJECTS = [(1, (2, 2, 2), (9, 8, 7)), (3, (12, 3, 1), (19, 10, 8)), (9, (0, 12, 0), (10, 23, 6)),
           (9, (11, 14, 0), (22, 22, 6)), (11, (20, 0, 0), (31, 7, 5)), (5, (24, 12, 6), (31, 23, 15)),
           (2, (4, 16, 8), (9, 21, 13)), (14, (14, 0, 9), (27, 11, 15)), (0, (0, 0, 0), (5, 5, 5)),
           (K1 - 1, (6, 6, 6), (12, 12, 12)), (6, (27, 18, 0), (31, 23, 4)), (4, (0, 0, 10), (3, 5, 15))]


def box_size():
    return tuple(int(np.ceil((h - l + 1) / 8.0)) * 8 for l, h in zip(MIN_C, MAX_C))


def synthetic(step, m):
    """One subnet's training output and labels, plain tensors (the test reads the same from the .npz)."""
    g = torch.Generator().manual_seed(100 * step + m)
    X, Y, Z = box_size()
    lo = torch.tensor(MIN_C)
    # mask rows: ~20 % of the box cells, plus every third cell of the x = 0 and x = X - 1 faces and of the z = Z - 1 face
    occ = torch.rand(X, Y, Z, generator=g) < 0.2
    occ[0, ::3, ::3], occ[-1, ::3, ::3], occ[::3, ::3, -1] = True, True, True
    cells = torch.nonzero(occ)
    vox_C = torch.cat([torch.zeros(len(cells), 1, dtype=torch.int32), (cells + lo).int()], 1)
    vox_F = torch.randn(len(cells), Q, generator=g) * 1.5 - 4.0
    query = torch.randn(1, Q, K1, generator=g)
    for q, (cls, a, b) in enumerate(OBJECTS):
        a = [v + int(torch.randint(-1, 2, (1,), generator=g)) for v in a]
        inside = ((cells >= torch.tensor(a)) & (cells <= torch.tensor(b))).all(1)
        vox_F[inside, q] += 7.0 + torch.rand(int(inside.sum()), generator=g) * 2
        query[0, q, cls] += 9.0
    if step == 0 and m == 1:
        query[0, :, K1 - 1] += 30.0                                       # no kept query
    # semantic rows: 60 % of the occupied cells (the others are labelled box cells without a row) plus rows outside
    # [min_C, max_C] (past max_C inside the box, and outside it)
    sem_cells = torch.cat([cells[torch.rand(len(cells), generator=g) < 0.6], torch.tensor([[X - 1, 0, 0], [-1, 3, 3], [5, Y + 2, 1], [3, 3, Z - 1], [40, 2, 2]])])
    sem_C = torch.cat([torch.zeros(len(sem_cells), 1, dtype=torch.int32), (sem_cells + lo).int()], 1)
    sem_F = torch.randn(len(sem_cells), K, generator=g)
    # ground truth: each kept object's box (jittered) with its class, a 255 slab, a missed instance, stuff 9 twice
    label = torch.zeros(X, Y, Z, dtype=torch.uint8)
    items = []
    for cls, a, b in OBJECTS:
        if cls in (0, K1 - 1):
            continue
        a = [max(0, v + int(torch.randint(-2, 3, (1,), generator=g))) for v in a]
        items.append((cls, a, b))
    items.append((7, (14, 18, 10), (18, 22, 14)))                         # missed
    masks = torch.zeros(len(items), X, Y, Z, dtype=torch.bool)
    for i, (cls, a, b) in enumerate(items):
        sl = tuple(slice(u, v + 1) for u, v in zip(a, b))
        masks[i][sl] = occ[sl]
        label[sl] = torch.where(occ[sl], torch.tensor(cls, dtype=torch.uint8), label[sl])
    sc = torch.stack([sem_cells[:, d].clamp(0, n - 1) for d, n in enumerate((X, Y, Z))], 1)
    lab_at = label[sc[:, 0], sc[:, 1], sc[:, 2]].long()                     # semantic logits lean to the label
    sem_F[torch.arange(len(sem_cells)), lab_at] += 2.5
    label[:, :, 3] = torch.where(torch.rand(X, Y, generator=g) < 0.7, torch.tensor(255, dtype=torch.uint8), label[:, :, 3])
    vox_F, sem_F = quantise(vox_F), quantise(sem_F)
    labels = torch.tensor([cls for cls, _, _ in items], dtype=torch.uint8)
    return {"vox_C": vox_C, "vox_F": vox_F, "query": query, "sem_C": sem_C, "sem_F": sem_F, "label": label,
            "labels": labels, "masks": masks}


def main():
    sys.path[:0] = [os.path.join(ROOT, "oracle", "shims"), os.path.join(ROOT, "compat"), "/root/reference", ROOT,
                    os.path.join(ROOT, "oracle"), os.path.join(ROOT, "oracle", "tools"), HERE]
    import MinkowskiEngine as ME
    import pasco.models.metrics as MET
    import pasco.models.net_panoptic_sparse as NPS
    import torch.nn.functional as F
    from pasco.loss.panoptic_quality import PQStat
    from pasco.models.helper import panoptic_inference
    from pasco.models.misc import compute_scene_size, prune_outside_coords
    Net = NPS.Net
    stub = types.SimpleNamespace(thing_ids=THING_IDS, n_classes=K, uncertainty_thresholds=[0.5])
    stub.evaluate_panoptic = types.MethodType(Net.evaluate_panoptic, stub)
    pq = [PQStat() for _ in range(M)]
    ssc = [MET.SSCMetrics(K) for _ in range(M)]
    min_C, max_C = torch.tensor(MIN_C), torch.tensor(MAX_C)
    arrays = {"min_C": min_C.numpy(), "max_C": max_C.numpy()}
    for step in range(STEPS):
        for m in range(M):
            d = synthetic(step, m)
            for k, v in d.items():
                arrays[f"s{step}m{m}_{k}"] = to_stored(k, v)
            # net_panoptic_sparse.py:398, 430-459, as Net.step runs them
            voxel_probs = ME.MinkowskiSigmoid()(ME.SparseTensor(d["vox_F"], d["vox_C"]))
            query_probs = F.softmax(d["query"], dim=-1)
            scene_size = compute_scene_size(min_C, max_C, scale=8).int()
            panop_out = panoptic_inference(voxel_probs, query_probs, overlap_threshold=OVERLAP,
                                           object_mask_threshold=OBJECT_MASK, thing_ids=THING_IDS, scene_size=scene_size,
                                           min_C=min_C, input_query_logit=False, input_voxel_logit=False)
            sem_logits = prune_outside_coords(ME.SparseTensor(d["sem_F"], d["sem_C"]), min_C, max_C)
            shape = torch.Size([1, K, scene_size[0], scene_size[1], scene_size[2]])
            sem_logits = sem_logits.dense(shape, min_coordinate=torch.IntTensor([*min_C]))[0].squeeze()
            sem_prob = F.softmax(sem_logits, dim=0)
            Net.evaluate_all(stub, ssc_confidence=sem_prob.max(dim=0)[0], i_infer=m, sem_prob=sem_prob,
                             panop_out=panop_out, semantic_label=d["label"].unsqueeze(0),
                             mask_labels=[{"labels": d["labels"], "masks": d["masks"]}], ssc_metrics=ssc[m],
                             pq_stat=pq[m], uncertainty_metrics=None, compute_uncertainty=False)
            cats = sorted(pq[m].pq_per_cat)
            tag = f"after{step}_m{m}"
            arrays[tag + "_pq_cats"] = np.array(cats, np.int64)
            arrays[tag + "_pq_fields"] = np.array([[float(pq[m][c].all_iou), float(pq[m][c].all_n), float(pq[m][c].iou),
                                                    pq[m][c].tp, pq[m][c].fp, pq[m][c].fn] for c in cats],
                                                  np.float64).reshape(-1, 6)
            arrays[tag + "_completion"] = np.array([ssc[m].completion_tp, ssc[m].completion_fp, ssc[m].completion_fn],
                                                   np.int64)
            arrays[tag + "_class_counts"] = np.stack([ssc[m].tps, ssc[m].fps, ssc[m].fns]).astype(np.int64)
            print(f"step {step} subnet {m}: {len(panop_out['segments_infos'][0])} segments, "
                  f"tp/fp/fn per cat {[(c, pq[m][c].tp, pq[m][c].fp, pq[m][c].fn) for c in cats]}, "
                  f"completion {arrays[tag + '_completion'].tolist()}")
    out = os.path.join(HERE, "step_eval_m2.npz")
    np.savez_compressed(out, **arrays)
    print("wrote", out)


if __name__ == "__main__":
    main()
