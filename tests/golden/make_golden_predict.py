"""Golden vectors for PascoNet.predict — BUILD CONTAINER ONLY: runs the reference's OWN Ensembler
(pasco/models/ensembler.py:20-187), panoptic_inference (helper.py:91-303) and Net.forward(return_ensemble=True)
(net_panoptic_sparse.py:210-310) from the upstream checkout on the CPU (MinkowskiEngine = the oracle shim).

    python tests/golden/make_golden_predict.py

(a) predict_post.npz — post-processing at the real shape: Q = 100 queries, M = 3 subnets of ~50 k rows under an identity
    pose, a flip + translation and a 7-degree rotation.  The inputs are not stored (they would be ~60 MB): scene_a()
    below rebuilds them from a seed on any machine (CPU torch RNG, no reference code) and the fixture keeps their
    checksums.  The scene reaches every branch: a stuff class predicted by two queries (merged), a query dropped by the
    overlap filter, queries dropped by the mean-IoU keep, rows dropped by the ensembled occupancy gate.  Stored per entry
    (M subnets, then the ensemble): the sorted rows, panoptic / semantic labels and vox_confidence at the rows, the
    segments (id, isthing, category, query, confidence, all_class_probs), ssc_pred / ssc_confidence as a dense subsample
    plus sums, and the Hungarian assignment of every matching step.
(b) predict_e2e.npz — end to end: the net_cfg1 scene at M = 2 (second subnet under the flip + translation pose), network
    calibrated as make_golden_infer.py does (the same running statistics as net_cfg1_infer_m2.npz), reference
    Net.forward(return_ensemble=True, test=True), then panoptic_inference on every entry as step_inference does.  Stored
    as summaries: row count / key sum of every entry, label histograms, segment tables, a row subsample, confidence
    percentiles, ssc sums.
A manifest (predict_manifest.json) lists the cases, thresholds and array names.
"""
import json
import math
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))

import numpy as np  # noqa: E402
import torch  # noqa: E402

Q_A, K, N_A = 100, 20, 50_000
THING_IDS = [1, 2, 3, 4, 5, 6, 7, 8]
THR_A = dict(overlap_threshold=0.4, object_mask_threshold=0.7, iou_threshold=0.2)
THR_B = dict(overlap_threshold=0.4, object_mask_threshold=0.05, iou_threshold=0.2)
# objects on a lattice (well separated): (class, half-size in cells); class 9 twice (stuff merge); object 12 is a
# larger copy of object 0 with another class and a lower class probability (wins only its rim: the overlap filter)
OBJECTS = [(1, 9), (2, 8), (9, 8), (3, 8), (9, 9), (10, 8), (4, 8), (5, 9), (11, 8), (6, 8), (12, 8), (7, 8)]
CENTRES = [(60 + 40 * (j % 4), 70 + 55 * (j // 4), 16) for j in range(12)]
SUBSAMPLE = 997


def poses():
    r = math.radians(7.0)
    flip = torch.tensor([[1.0, 0, 0, 0.4], [0, -1.0, 0, -0.6], [0, 0, 1.0, 0], [0, 0, 0, 1.0]])
    rot = torch.tensor([[math.cos(r), -math.sin(r), 0, 0.0], [math.sin(r), math.cos(r), 0, 0.2], [0, 0, 1.0, 0],
                        [0, 0, 0, 1.0]], dtype=torch.float32)
    return [torch.eye(4), flip, rot]


def _transform(coords, T):
    """transform_utils.transform (restated: the inputs must be rebuildable without the reference)."""
    lo = torch.tensor([0.0, -25.6, -2.0]).view(1, 3)
    pts = coords.float() * 0.2 + 0.2 / 2 + lo
    hom = torch.cat([pts, torch.ones(pts.shape[0], 1)], 1)
    new = (T @ hom.t()).t()[:, :3]
    return torch.round((new - lo - 0.2 / 2) / 0.2).int()


def scene_a(seed=0, M=3, Q=Q_A, n=N_A):
    """Synthetic predictions of M subnets: 12 box objects + 1 overlap-filter query, noise queries that no two subnets
    agree on (dropped by the mean-IoU keep), semantic logits with every 7th row predicted empty (occupancy gate).
    Returns (preds, sems, Ts) with coords [N, 3] int in each subnet's frame."""
    g = torch.Generator().manual_seed(seed)
    Ts = poses()[:M]
    base = torch.stack([torch.randint(30, 220, (n,), generator=g), torch.randint(40, 215, (n,), generator=g),
                        torch.randint(2, 30, (n,), generator=g)], 1)
    base = torch.unique(base, dim=0)
    centres = torch.tensor(CENTRES, dtype=torch.float32)
    half = torch.tensor([h for _, h in OBJECTS] + [11], dtype=torch.float32)
    centres = torch.cat([centres, centres[:1]], 0)                  # query 12: the larger copy of object 0
    classes = [c for c, _ in OBJECTS] + [3]
    preds, sems = [], []
    for m in range(M):
        c = torch.unique(_transform(base, Ts[m]).long(), dim=0)
        back = _transform(c, torch.inverse(Ts[m])).float()
        d = (back[:, None, :] - centres[None]).abs().amax(-1)      # [n, 13] box distance
        logits = -8.0 + 1.5 * torch.randn(c.shape[0], Q, generator=g)
        perm = torch.randperm(Q, generator=g)
        for j in range(13):
            logits[:, perm[j]] = 3.0 * (half[j] - d[:, j]) + 0.3 * torch.randn(c.shape[0], generator=g)
        ql = torch.randn(1, Q, K + 1, generator=g)
        for j in range(13):
            ql[0, perm[j], classes[j]] += 7.0 if j < 12 else 4.0
        sem = torch.randn(c.shape[0], K, generator=g)
        rows = torch.arange(c.shape[0])
        sem[rows, 1 + rows % (K - 1)] += 2.0
        sem[::7, 0] += 8.0
        preds.append({"voxel_logits": (logits, c), "query_logits": ql})
        sems.append((sem, c))
    return preds, sems, Ts


def checksums(preds, sems):
    out = []
    for p, (s, sc) in zip(preds, sems):
        lg, c = p["voxel_logits"]
        out += [float(lg.double().sum()), float(c.double().sum()), float(p["query_logits"].double().sum()),
                float(s.double().sum()), float(sc.double().sum())]
    return np.array(out)


def _lin(C):
    C = C.long()
    return (C[:, 0] * 256 + C[:, 1]) * 32 + C[:, 2]


def _entries(ens, panoptic_inference, preds_ref, sem_denses, Ts, thr):
    """The reference's ensemble + panoptic_inference on every entry → per entry dict of sparse outputs."""
    out = ens.ensemble_panop(preds_ref, sem_denses, (256, 256, 32), Ts, iou_threshold=thr["iou_threshold"])
    res = []
    for o, sd in zip(out, sem_denses):
        r = panoptic_inference(o["voxel_probs"], o["query_probs"], overlap_threshold=thr["overlap_threshold"],
                               object_mask_threshold=thr["object_mask_threshold"], thing_ids=THING_IDS,
                               min_C=torch.tensor([0, 0, 0]), scene_size=(256, 256, 32), input_query_logit=False,
                               input_voxel_logit=False)
        C = o["voxel_probs"].C[:, 1:].long()
        lin = _lin(C)
        order = torch.argsort(lin)
        at = lambda v: v[0][C[:, 0], C[:, 1], C[:, 2]][order]                # noqa: E731
        flat = sd.reshape(sd.shape[0], -1)
        res.append({"lin": lin[order], "pan": r["panoptic_seg_sparses"][0][order], "sem": at(r["semantic_seg_denses"]),
                    "conf": at(r["vox_confidence_denses"]), "segments": r["segments_infos"][0],
                    "ssc_pred": flat.argmax(0), "ssc_conf": flat.max(0)[0], "n_queries": o["query_probs"].shape[1]})
    return res


def _store(arrays, tag, i, e, full_rows):
    arrays[f"{tag}{i}_n"] = np.array([e["lin"].numel()])
    arrays[f"{tag}{i}_linsum"] = np.array([int(e["lin"].sum())])
    sel = slice(None) if full_rows else slice(None, None, 7)
    arrays[f"{tag}{i}_lin"] = e["lin"][sel].numpy().astype(np.int32)
    arrays[f"{tag}{i}_pan"] = e["pan"][sel].numpy().astype(np.int32)
    arrays[f"{tag}{i}_sem"] = e["sem"][sel].numpy().astype(np.int32)
    arrays[f"{tag}{i}_conf"] = e["conf"][sel].numpy().astype(np.float32)
    arrays[f"{tag}{i}_pan_hist"] = np.bincount(e["pan"].numpy(), minlength=64)[:64]
    arrays[f"{tag}{i}_sem_hist"] = np.bincount(e["sem"].numpy(), minlength=21)[:21]
    arrays[f"{tag}{i}_conf_sum"] = np.array([float(e["conf"].double().sum())])
    arrays[f"{tag}{i}_conf_pct"] = np.percentile(e["conf"].numpy(), [50, 90, 99]) if e["conf"].numel() else np.zeros(3)
    segs = e["segments"]
    arrays[f"{tag}{i}_segments"] = np.array([[s["id"], int(s["isthing"]), s["category_id"], s["query_id"]] for s in segs],
                                            dtype=np.int64).reshape(-1, 4)
    arrays[f"{tag}{i}_seg_conf"] = np.array([s["confidence"] for s in segs], dtype=np.float64)
    arrays[f"{tag}{i}_seg_probs"] = np.stack([s["all_class_probs"].numpy() for s in segs]).astype(np.float32) \
        if segs else np.zeros((0, K + 1), np.float32)
    arrays[f"{tag}{i}_n_queries"] = np.array([e["n_queries"]])
    arrays[f"{tag}{i}_ssc_pred_sub"] = e["ssc_pred"][::SUBSAMPLE].numpy().astype(np.int32)
    arrays[f"{tag}{i}_ssc_conf_sub"] = e["ssc_conf"][::SUBSAMPLE].numpy().astype(np.float32)
    arrays[f"{tag}{i}_ssc_sums"] = np.array([float(e["ssc_conf"].double().sum()), float((e["ssc_pred"] != 0).sum()),
                                             float(e["ssc_pred"].double().sum())])


def main():
    sys.path[:0] = [os.path.join(ROOT, "oracle", "shims"), os.path.join(ROOT, "compat"), "/root/reference", ROOT,
                    os.path.join(ROOT, "oracle"), os.path.join(ROOT, "oracle", "tools"), HERE]
    torch.set_num_threads(os.cpu_count())
    import MinkowskiEngine as ME
    import pasco.models.ensembler as ENS
    from pasco.models.helper import panoptic_inference
    matches = []
    orig = ENS.find_matching_indices_v2

    def recording(*a, **k):
        r = orig(*a, **k)
        matches.append((np.asarray(r[0]), np.asarray(r[1])))
        return r
    ENS.find_matching_indices_v2 = recording
    bc = lambda c: ME.utils.batched_coordinates([c])   # noqa: E731
    manifest = {"a": {"Q": Q_A, "M": 3, "thresholds": THR_A, "subsample": SUBSAMPLE}, "b": {}}

    # (a) post-processing at the real shape
    preds, sems, Ts = scene_a()
    ens = ENS.Ensembler()
    sem_denses = ens.ensemble_sem_compl({1: [ME.SparseTensor(f, bc(c)) for f, c in sems]}, Ts)
    ref_preds = [{"voxel_logits": ME.SparseTensor(p["voxel_logits"][0], bc(p["voxel_logits"][1])),
                  "query_logits": p["query_logits"]} for p in preds]
    res = _entries(ens, panoptic_inference, ref_preds, sem_denses, Ts, THR_A)
    arrays = {"input_checksums": checksums(preds, sems)}
    for i, e in enumerate(res):
        _store(arrays, "a", i, e, full_rows=True)
    for s, (ai, bi) in enumerate(matches):
        arrays[f"a_match{s}"] = np.stack([ai, bi]).astype(np.int32)
    ensm = res[-1]
    assert ensm["n_queries"] < Q_A, "the mean-IoU keep must drop queries"
    assert int(((ensm["pan"] != 0) & (ensm["sem"] == 0)).sum()) > 0, "a stuff class must merge"
    assert (ensm["lin"].numel() < res[0]["lin"].numel() + res[1]["lin"].numel()), "the occupancy gate must drop rows"
    np.savez_compressed(os.path.join(HERE, "predict_post.npz"), **arrays)
    manifest["a"]["arrays"] = sorted(arrays)
    print("(a)", {k: v.tolist() for k, v in arrays.items() if k.endswith(("_n", "_n_queries"))},
          [len(e["segments"]) for e in res])

    # (b) end to end on the net_cfg1 scene at M = 2
    from make_golden_infer import GRID, OCC, SEED, calibrated_net
    from run_reference_on_oracle import forward
    from pasco_b200.synthetic import make_scene
    matches.clear()
    net = calibrated_net(2, GRID, OCC)
    batch = make_scene(GRID, OCC, 2, seed=SEED)
    Tb = poses()[:2]
    batch["Ts"] = Tb
    net.ensembler = ENS.Ensembler()
    with torch.no_grad():
        _rp = torch.randperm
        torch.randperm = lambda n, device=None, **k: _rp(n, **k)
        try:
            ic, iff = net.feat(batch["in_feats"], batch["in_coords"])
        finally:
            torch.randperm = _rp
        in_feat = net.augmenter.merge(ME.SparseTensor(iff, ic.int()))
        ssc_confs, sem_denses, panop = net(in_feat, 1, batch["sem_labels"], global_min_coords=batch["global_min_Cs"],
                                           global_max_coords=batch["global_max_Cs"], min_Cs=batch["min_Cs"],
                                           max_Cs=batch["max_Cs"], Ts=Tb, is_predict_panop=True, return_ensemble=True,
                                           test=True)
    arrays = {}
    for i, (o, sd, sc) in enumerate(zip(panop, sem_denses, ssc_confs)):
        r = panoptic_inference(o["voxel_probs"], o["query_probs"], overlap_threshold=THR_B["overlap_threshold"],
                               object_mask_threshold=THR_B["object_mask_threshold"], thing_ids=THING_IDS,
                               min_C=torch.tensor([0, 0, 0]), scene_size=(256, 256, 32), input_query_logit=False,
                               input_voxel_logit=False)
        C = o["voxel_probs"].C[:, 1:].long()
        lin = _lin(C)
        order = torch.argsort(lin)
        at = lambda v: v[0][C[:, 0], C[:, 1], C[:, 2]][order]                # noqa: E731
        flat = sd.reshape(sd.shape[0], -1)
        assert torch.equal(sc.reshape(-1), flat.max(0)[0])
        e = {"lin": lin[order], "pan": r["panoptic_seg_sparses"][0][order], "sem": at(r["semantic_seg_denses"]),
             "conf": at(r["vox_confidence_denses"]), "segments": r["segments_infos"][0], "ssc_pred": flat.argmax(0),
             "ssc_conf": flat.max(0)[0], "n_queries": o["query_probs"].shape[1]}
        _store(arrays, "b", i, e, full_rows=False)
    for s, (ai, bi) in enumerate(matches):
        arrays[f"b_match{s}"] = np.stack([ai, bi]).astype(np.int32)
    np.savez_compressed(os.path.join(HERE, "predict_e2e.npz"), **arrays)
    manifest["b"] = {"grid": list(GRID), "occ": OCC, "seed": SEED, "M": 2, "thresholds": THR_B,
                     "running_stats_from": "net_cfg1_infer_m2.npz", "arrays": sorted(arrays)}
    print("(b)", {k: v.tolist() for k, v in arrays.items() if k.endswith(("_n", "_n_queries"))})
    json.dump(manifest, open(os.path.join(HERE, "predict_manifest.json"), "w"), indent=0)


if __name__ == "__main__":
    main()
