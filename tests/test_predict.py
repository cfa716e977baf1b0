"""PascoNet.predict and its post-processing kernels (csrc/panoptic.cu, pasco_b200/predict.py) against the torch
restatement of the reference's Ensembler and panoptic_inference (pasco_b200/ensemble.py, itself pinned to the reference by
tests/test_ensemble.py), on synthetic M-subnet predictions at Q = 24, 100, 200 and 600 queries under an identity pose, a
flip + translation and a 7-degree rotation.

  * CPU: the torch confidence outputs against a literal per-query restatement of helper.py:135-263, the new entry points'
    header and ctypes signatures, predict's training-mode refusal;
  * GPU: every stage (warp, activation + column sums, soft IoU, merge, semantic ensemble, panoptic passes) against
    ensemble.py — integers exactly, floats to 1e-6 relative, the IoU also against an fp64 recompute — plus edge cases,
    bit-identical repeat calls, host synchronisations independent of Q, and PascoNet.predict end to end;
  * against fixtures the reference's own code produced (tests/golden/make_golden_predict.py): (a) its Ensembler and
    panoptic_inference at Q = 100, M = 3 — the torch function on the CPU and predict's post-processing on the GPU, rows,
    labels, segments and Hungarian assignments exactly, confidences to 1e-5 — and (b) its Net.forward(return_ensemble=True)
    + panoptic_inference on the net_cfg1 scene at M = 2, against PascoNet.predict with the eval tests' near-tie tolerance.
"""
import collections
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
import make_golden_predict as GP  # noqa: E402  (scene_a rebuilds fixture (a)'s inputs; the reference is not imported)
import parity  # noqa: E402

FIX_A = np.load(os.path.join(GOLD, "predict_post.npz"))
FIX_B = np.load(os.path.join(GOLD, "predict_e2e.npz"))
MANIFEST = json.load(open(os.path.join(GOLD, "predict_manifest.json")))

K = 20
SIZE = (256, 256, 32)
CELLS = SIZE[0] * SIZE[1] * SIZE[2]
THR = dict(overlap_threshold=0.5, object_mask_threshold=0.2, iou_threshold=0.2)
# object classes: things 1-8, stuff class 9 predicted by two objects (merged), stuff 10-12 once each
OBJ_CLASSES = [1, 2, 9, 3, 9, 10, 4, 5, 11, 6, 12, 7]


def _poses():
    r = math.radians(7.0)
    flip = torch.tensor([[1.0, 0, 0, 0.4], [0, -1.0, 0, -0.6], [0, 0, 1.0, 0], [0, 0, 0, 1.0]])
    rot = torch.tensor([[math.cos(r), -math.sin(r), 0, 0.0], [math.sin(r), math.cos(r), 0, 0.2], [0, 0, 1.0, 0],
                        [0, 0, 0, 1.0]], dtype=torch.float32)
    return [torch.eye(4), flip, rot]


def _scene(Q, M=3, seed=0, n=6000, dev="cpu", far=()):
    """M subnets looking at 12 blobs under their poses; subnet m's queries are a permutation of the objects.  Subnets in
    `far` see the scene moved outside the reference grid (no voxel inside)."""
    from pasco_b200 import ensemble as E
    g = torch.Generator().manual_seed(seed)
    Ts = _poses()[:M]
    base = torch.stack([torch.randint(40, 200, (n,), generator=g), torch.randint(40, 200, (n,), generator=g),
                        torch.randint(2, 30, (n,), generator=g)], 1)
    base = torch.unique(base, dim=0)
    centres = base[torch.randperm(base.shape[0], generator=g)[:12]].float()
    n_obj = min(12, Q)
    preds, sems = [], []
    for m in range(M):
        c = torch.unique(E._transform(base, Ts[m]).long(), dim=0)
        back = E._transform(c, torch.inverse(Ts[m])).float()
        d = (back[:, None, :] - centres[None]).abs().amax(-1)
        logits = torch.full((c.shape[0], Q), -9.0)
        logits += 0.5 * torch.randn(c.shape[0], Q, generator=g)
        perm = torch.randperm(Q, generator=g)
        for j in range(n_obj):
            logits[:, perm[j]] = 7.0 - 0.6 * d[:, j] + 0.3 * torch.randn(c.shape[0], generator=g)
        ql = torch.randn(1, Q, K + 1, generator=g)
        for j in range(n_obj):
            ql[0, perm[j], OBJ_CLASSES[j]] += 6.0
        sem = torch.randn(c.shape[0], K, generator=g)
        sem[torch.arange(c.shape[0]), 1 + (torch.arange(c.shape[0]) % (K - 1))] += 2.0
        sem[::7, 0] += 6.0                                           # empty-class rows: the occupancy gate drops them
        if m in far:
            c = c + 1000
        preds.append({"voxel_logits": (logits.to(dev), c.to(dev)), "query_logits": ql.to(dev)})
        sems.append((sem.to(dev), c.to(dev)))
    return preds, sems, Ts


def _literal_panoptic(voxel_probs, query_probs, overlap_threshold, object_mask_threshold, thing_ids, vox_occ=0.3):
    """helper.py:135-263, the per-query loop as written upstream (one batch item, sparse outputs)."""
    n_classes = query_probs.shape[-1] - 1
    probs, labels = query_probs.max(-1)
    keep = labels.ne(0) & labels.ne(n_classes) & (probs > object_mask_threshold)
    fp, fc, fall = probs[keep], labels[keep], query_probs[keep]
    fids = torch.arange(keep.shape[0])[keep]
    masks = voxel_probs[:, keep]
    norm = masks / (masks.sum(1, keepdim=True) + 1e-8)
    comb = fp.view(1, -1) * masks
    N = masks.shape[0]
    pan = torch.zeros(N, dtype=torch.int32)
    sem = torch.zeros(N, dtype=torch.int32)
    conf = torch.zeros(N)
    infos, cur_id = [], 0
    if masks.shape[1] != 0:
        _, cur = comb.max(1)
        stuff = {}
        for k in range(fc.shape[0]):
            pc, qp = fc[k].item(), fp[k].item()
            isthing = pc in thing_ids
            mask = (cur == k) & (masks[:, k] >= vox_occ)
            ma, oa = mask.sum().item(), (masks[:, k] >= vox_occ).sum().item()
            if ma > 0 and oa > 0:
                if ma / oa < overlap_threshold:
                    continue
                if not isthing:
                    if int(pc) in stuff:
                        pan[mask] = stuff[int(pc)]
                        continue
                    stuff[int(pc)] = cur_id + 1
                cur_id += 1
                pan[mask] = cur_id
                sem[mask] = pc
                conf[mask] = norm[mask, k]
                infos.append({"id": cur_id, "isthing": bool(isthing), "category_id": int(pc), "query_id": fids[k].item(),
                              "confidence": qp, "all_class_probs": fall[k]})
    return pan, sem, conf, infos


def _same_infos(a, b, atol=0.0):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert {k: x[k] for k in ("id", "isthing", "category_id", "query_id")} == \
               {k: y[k] for k in ("id", "isthing", "category_id", "query_id")}
        assert abs(x["confidence"] - y["confidence"]) <= atol
        assert torch.allclose(x["all_class_probs"].cpu(), y["all_class_probs"].cpu(), atol=atol, rtol=0)


# ------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------
def test_confidence_outputs_match_the_literal_reference_loop():
    from pasco_b200 import ensemble as E
    preds, sems, Ts = _scene(24)
    sem_denses = E.ensemble_sem_compl(sems, Ts)
    out = E.ensemble_panop(preds, sem_denses, Ts, iou_threshold=0.2)
    for o in out:
        prob, _ = o["voxel_probs"]
        qp = o["query_probs"][0]
        for thr in (THR, dict(overlap_threshold=0.4, object_mask_threshold=0.7)):
            pan, sem, conf, infos = E.panoptic_inference_with_confidence(
                prob, qp, thr["overlap_threshold"], thr["object_mask_threshold"], [1, 2, 3, 4, 5, 6, 7, 8])
            rp, rs, rc, ri = _literal_panoptic(prob, qp, thr["overlap_threshold"], thr["object_mask_threshold"],
                                               [1, 2, 3, 4, 5, 6, 7, 8])
            assert torch.equal(pan, rp) and torch.equal(sem, rs) and torch.equal(conf, rc)
            _same_infos(infos, ri)
            p0, s0, i0 = E.panoptic_inference(prob, qp, thr["overlap_threshold"], thr["object_mask_threshold"],
                                              [1, 2, 3, 4, 5, 6, 7, 8])
            assert torch.equal(p0, pan) and torch.equal(s0, sem) and len(i0) == len(infos)
    # two queries of one stuff class: the second merges into the first segment and keeps semantic 0 and confidence 0
    q = torch.full((3, 21), 1e-3)
    q[:2, 12], q[2, 3] = 0.9, 0.9
    v = torch.zeros(60, 3)
    v[:20, 0], v[20:40, 1], v[40:, 2] = 0.9, 0.8, 0.7
    pan, sem, conf, infos = E.panoptic_inference_with_confidence(v, q, 0.5, 0.2, [1, 2, 3])
    rp, rs, rc, ri = _literal_panoptic(v, q, 0.5, 0.2, [1, 2, 3])
    assert torch.equal(pan, rp) and torch.equal(sem, rs) and torch.equal(conf, rc)
    _same_infos(infos, ri)
    assert pan[20:40].eq(1).all() and sem[20:40].eq(0).all() and conf[20:40].eq(0).all() and conf[:20].gt(0.99).all()


def test_predict_refuses_training_mode():
    from pasco_b200.net3d import PascoNet
    net = PascoNet(n_infers=1).train()
    with pytest.raises(RuntimeError, match="eval"):
        net.predict([], [], None, None, None, None)


# ------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------
def _torch_entries(preds, sems, Ts, thr):
    from pasco_b200 import ensemble as E
    sem_denses = E.ensemble_sem_compl(sems, Ts)
    out = E.ensemble_panop(preds, sem_denses, Ts, iou_threshold=thr["iou_threshold"])
    res = []
    for o, sd in zip(out, sem_denses):
        prob, lin = o["voxel_probs"]
        order = torch.argsort(lin)
        prob, lin = prob[order], lin[order]
        qp = o["query_probs"][0]
        pan, sem, conf, infos = E.panoptic_inference_with_confidence(prob, qp, thr["overlap_threshold"],
                                                                     thr["object_mask_threshold"], [1, 2, 3, 4, 5, 6, 7, 8])
        res.append(dict(lin=lin, prob=prob, qp=qp, pan=pan, sem=sem, conf=conf, infos=infos, sem_dense=sd))
    return res


def _near_half_cells(T):
    """Cells whose transformed coordinate lies within 1e-5 of a .5 rounding boundary (fp64 recompute)."""
    g = torch.stack(torch.meshgrid(*[torch.arange(s, dtype=torch.float64) for s in SIZE], indexing="ij"), -1).view(-1, 3)
    lo = torch.tensor([0.0, -25.6, -2.0], dtype=torch.float64)
    p = g * 0.2 + 0.1 + lo
    v = (p @ T[:3, :3].double().t() + T[:3, 3].double() - lo - 0.1) / 0.2
    return ((v - v.floor() - 0.5).abs() < 1e-5).any(1)


def _check_entries(got, ref, Q):
    for e, r in zip(got, ref):
        assert torch.equal(e["lin"].cpu(), r["lin"].cpu()), "row set"
        assert e["query_probs"].shape[0] == r["prob"].shape[1]
        torch.testing.assert_close(e["query_probs"], r["qp"], rtol=1e-6, atol=1e-7)
        assert torch.equal(e["panoptic_seg"], r["pan"]) and torch.equal(e["semantic_seg"], r["sem"])
        torch.testing.assert_close(e["vox_confidence"], r["conf"], rtol=1e-5, atol=1e-6)
        _same_infos(e["segments_info"], r["infos"], atol=1e-6)
        flat = r["sem_dense"].reshape(K, -1)
        from pasco_b200.predict import to_dense
        assert torch.equal(to_dense(e, "ssc_pred").view(-1).long(), flat.argmax(0))
        torch.testing.assert_close(to_dense(e, "ssc_confidence").view(-1), flat.max(0)[0], rtol=1e-6, atol=1e-7)
        dpan = to_dense(e, "panoptic_seg").view(-1)
        assert torch.equal(dpan[e["lin"]], e["panoptic_seg"]) and int(dpan.ne(0).sum()) == int(e["panoptic_seg"].ne(0).sum())


@pytest.mark.gpu
@pytest.mark.parametrize("Q", [24, 100, 200, 600])
def test_postprocess_matches_the_torch_ensemble(Q):
    from pasco_b200 import ensemble as E, ops, predict as P
    dev = torch.device("cuda")
    preds, sems, Ts = _scene(Q, dev=dev)
    # warp: the cell sets are exact except, possibly, at cells within 1e-5 of a rounding boundary
    for m, T in enumerate(Ts):
        logits, coords = preds[m]["voxel_logits"]
        lin, cell, src = P.warp(coords, T)
        rprob, rlin = E.warp_to_reference_frame(torch.sigmoid(logits), coords, T)
        near = _near_half_cells(T)
        print(f"pose {m}: {int(near.sum())} cells within 1e-5 of a .5 boundary")
        diff = np.setxor1d(lin.cpu().numpy(), rlin.cpu().numpy())
        assert near[torch.as_tensor(diff, dtype=torch.long)].all()
        assert len(diff) == 0 or int(near.sum()) > 0
        assert torch.equal(cell[lin.long()].cpu(), torch.arange(lin.shape[0], dtype=torch.int32))
        prob, planes, colsum, nz = ops.mask_rows_sigmoid(logits, src)
        order = torch.argsort(rlin)
        torch.testing.assert_close(prob, rprob[order], rtol=1e-6, atol=1e-7)
        torch.testing.assert_close(colsum.double(), rprob.double().sum(0), rtol=1e-5, atol=1e-4)
        hi, lo = planes
        assert hi.shape[1] == ops.plane_cols(Q) and not hi[:, Q:].float().any()
        assert torch.equal(nz.bool(), prob.ne(0).any(1))
        if m == 0:
            anchor = (prob, planes, colsum, lin, cell)
        elif m == 1:   # soft IoU against an fp64 recompute (bf16x3 products: ~2^-16 relative)
            ap, apl, acs, alin, acell = anchor
            gated = ops.soft_iou(ap, apl, acs, prob, planes, colsum, ops.lookup_rows(acell, lin), 0.2)
            iou64 = E.soft_iou(ap.double(), alin.long(), prob.double(), lin.long(), CELLS)
            ref = torch.where(iou64 > 0.2, iou64, torch.zeros_like(iou64))
            near_thr = (iou64 - 0.2).abs() < 1e-4
            assert ((gated.double() - ref).abs()[~near_thr] <= 5e-5 * ref.abs().clamp(min=1.0)[~near_thr]).all()
            assert float(ref.max()) > 0.5
    # the whole post-processing against ensemble.py on the same outputs
    matches = []
    got = P.postprocess(preds, sems, Ts, matches=matches, **THR)
    ref = _torch_entries(preds, sems, Ts, THR)
    assert len(got) == 4
    _check_entries(got, ref, Q)
    ens = got[-1]
    assert ens["query_probs"].shape[0] < Q, "the mean-IoU keep drops queries"
    assert len(ens["segments_info"]) >= 4
    # square assignments: every anchor query is matched (the ensembled query probabilities above pin which)
    assert len(matches) == 2
    for ai, bi in matches:
        assert np.array_equal(ai, np.arange(Q)) and sorted(bi.tolist()) == list(range(Q))


@pytest.mark.gpu
def test_postprocess_edge_cases():
    from pasco_b200 import ensemble as E, ops, predict as P
    dev = torch.device("cuda")
    # M = 1: two entries, no matching
    preds, sems, Ts = _scene(100, M=1, dev=dev)
    matches = []
    got = P.postprocess(preds, sems, Ts, matches=matches, **THR)
    assert len(got) == 2 and matches == []
    _check_entries(got, _torch_entries(preds, sems, Ts, THR), 100)
    # a subnet with no voxel inside the grid
    preds, sems, Ts = _scene(100, M=3, dev=dev, far=(2,))
    got = P.postprocess(preds, sems, Ts, **THR)
    _check_entries(got, _torch_entries(preds, sems, Ts, THR), 100)
    assert got[2]["lin"].numel() == 0 and got[2]["segments_info"] == [] and got[2]["ssc_lin"].numel() == 0
    # no kept query
    got = P.postprocess(preds, sems, Ts, overlap_threshold=0.5, object_mask_threshold=0.999, iou_threshold=0.2)
    assert all(e["segments_info"] == [] and not e["panoptic_seg"].any() and not e["vox_confidence"].any() for e in got)
    # N = 0
    pan, sem, conf, rec = ops.panoptic(torch.zeros(0, 5, device=dev), torch.softmax(torch.randn(5, 21, device=dev), -1),
                                       0.5, 0.0, [1, 2])
    assert pan.numel() == 0 and int(rec[0]) == 0
    # all stuff: every kept query of one stuff class → one segment; all-zero rows (argmax ties at the lowest index)
    q = torch.full((6, 21), 1e-3, device=dev)
    q[:, 12] = 0.9
    v = torch.rand(4000, 6, device=dev)
    v[::5] = 0.0
    for probs in (v, torch.zeros(300, 6, device=dev)):
        pan, sem, conf, rec = ops.panoptic(probs, q, 0.0, 0.2, [1, 2, 3])
        rp, rs, rc, ri = E.panoptic_inference_with_confidence(probs, q, 0.0, 0.2, [1, 2, 3])
        assert torch.equal(pan, rp) and torch.equal(sem, rs)
        torch.testing.assert_close(conf, rc, rtol=1e-5, atol=1e-6)
        assert int(rec[0]) == len(ri) <= 1


@pytest.mark.gpu
def test_postprocess_is_bit_identical_across_calls():
    from pasco_b200 import predict as P
    preds, sems, Ts = _scene(100, dev=torch.device("cuda"))
    a, b = (P.postprocess(preds, sems, Ts, **THR) for _ in range(2))
    for x, y in zip(a, b):
        for k in ("lin", "panoptic_seg", "semantic_seg", "vox_confidence", "ssc_lin", "ssc_pred", "ssc_confidence",
                  "query_probs"):
            assert torch.equal(x[k], y[k]), k
        assert [(s["id"], s["query_id"], s["confidence"]) for s in x["segments_info"]] == \
               [(s["id"], s["query_id"], s["confidence"]) for s in y["segments_info"]]


@pytest.mark.gpu
def test_host_synchronisations_do_not_grow_with_the_query_count():
    from pasco_b200 import predict as P
    counts = {}
    for Q in (100, 200):
        preds, sems, Ts = _scene(Q, dev=torch.device("cuda"))
        P.postprocess(preds, sems, Ts, **THR)                       # warm-up (module loads, pools)
        torch.cuda.synchronize()
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            torch.cuda.set_sync_debug_mode("warn")
            try:
                P.postprocess(preds, sems, Ts, **THR)
            finally:
                torch.cuda.set_sync_debug_mode("default")
        sites = collections.Counter(f"{os.path.basename(x.filename)}:{x.lineno}" for x in w      # the engine's own calls
                                    if "synchroniz" in str(x.message) and f"{os.sep}pasco_b200{os.sep}" in x.filename)
        counts[Q] = sum(sites.values())
        print(f"Q = {Q}: host synchronisations by call site {dict(sites)}")
    assert counts[100] == counts[200] > 0


@pytest.mark.gpu
def test_pasconet_predict_end_to_end():
    """PascoNet.predict at M = 2 (second subnet under a flip + translation) against the forward's own outputs run through
    ensemble.py, and the dense volumes of to_dense."""
    from pasco_b200 import ops
    from pasco_b200.net3d import PascoNet
    from pasco_b200.synthetic import make_scene
    dev = torch.device("cuda")
    ops.set_precision("fp32")
    torch.manual_seed(0)
    net = PascoNet(n_infers=2).to(dev).eval()
    sc = make_scene((128, 128, 16), 0.05, 2, seed=0)
    args = ([t.to(dev) for t in sc["in_feats"]], [t.to(dev) for t in sc["in_coords"]], sc["global_min_Cs"],
            sc["global_max_Cs"], sc["min_Cs"], sc["max_Cs"])
    Ts = _poses()[:2]
    with pytest.raises(RuntimeError):
        net.train().predict(*args, Ts)
    net.eval()
    got = net.predict(*args, Ts, **THR)
    with torch.no_grad():
        ret = net(*args, predict_panop=True, test=True)
    preds = [{"voxel_logits": (p["voxel_logits"].F, p["voxel_logits"].C[:, 1:]), "query_logits": p["query_logits"]}
             for p in ret["panop_predictions"]]
    sems = [(s.F, s.C[:, 1:]) for s in ret["sem_logits_at_scales"][1]]
    assert len(got) == 3
    _check_entries(got, _torch_entries(preds, sems, Ts, THR), 100)
    assert got[0]["lin"].numel() > 0 and got[1]["lin"].numel() > 0


# ------------------------------------------------------------------------------------------------
# against the reference's own Ensembler / panoptic_inference / Net.forward (tests/golden/make_golden_predict.py)
# ------------------------------------------------------------------------------------------------
def _scene_a(dev):
    preds, sems, Ts = GP.scene_a()
    mv = lambda t: t.to(dev)  # noqa: E731
    preds = [{"voxel_logits": tuple(map(mv, p["voxel_logits"])), "query_logits": mv(p["query_logits"])} for p in preds]
    return preds, [tuple(map(mv, s)) for s in sems], Ts


def _check_fixture_a(i, lin, pan, sem, conf, infos, ssc_pred_dense, ssc_conf_dense, n_queries):
    """Entry i of fixture (a): rows, labels and segments exactly; confidences within 1e-5."""
    z = FIX_A
    assert np.array_equal(lin.cpu().numpy(), z[f"a{i}_lin"]), f"rows of entry {i}"
    assert np.array_equal(pan.cpu().numpy(), z[f"a{i}_pan"]), f"panoptic labels of entry {i}"
    assert np.array_equal(sem.cpu().numpy(), z[f"a{i}_sem"]), f"semantic labels of entry {i}"
    assert np.allclose(conf.cpu().numpy(), z[f"a{i}_conf"], rtol=0, atol=1e-5), f"vox_confidence of entry {i}"
    got = np.array([[s["id"], int(s["isthing"]), s["category_id"], s["query_id"]] for s in infos], dtype=np.int64)
    assert np.array_equal(got.reshape(-1, 4), z[f"a{i}_segments"]), f"segments of entry {i}"
    assert np.allclose([s["confidence"] for s in infos], z[f"a{i}_seg_conf"], rtol=0, atol=1e-5)
    probs = np.stack([s["all_class_probs"].cpu().numpy() for s in infos]) if infos else np.zeros((0, 21))
    assert np.allclose(probs, z[f"a{i}_seg_probs"], rtol=0, atol=1e-5)
    assert int(z[f"a{i}_n_queries"][0]) == n_queries
    sp, sc = ssc_pred_dense.reshape(-1).cpu(), ssc_conf_dense.reshape(-1).cpu()
    assert np.array_equal(sp[::GP.SUBSAMPLE].numpy(), z[f"a{i}_ssc_pred_sub"])
    assert np.allclose(sc[::GP.SUBSAMPLE].numpy(), z[f"a{i}_ssc_conf_sub"], rtol=0, atol=1e-5)
    ref = z[f"a{i}_ssc_sums"]
    assert int((sp != 0).sum()) == int(ref[1]) and int(sp.double().sum()) == int(ref[2])
    assert abs(float(sc.double().sum()) - ref[0]) <= 1e-5 * ref[0]


def test_predict_fixture_manifest_and_inputs():
    """The manifest lists every array of both fixtures, and scene_a rebuilds fixture (a)'s inputs bit for bit."""
    assert sorted(FIX_A.files) == MANIFEST["a"]["arrays"] and sorted(FIX_B.files) == MANIFEST["b"]["arrays"]
    assert MANIFEST["a"]["Q"] == 100 and MANIFEST["a"]["M"] == 3 and MANIFEST["b"]["M"] == 2
    preds, sems, _ = GP.scene_a()
    assert np.array_equal(GP.checksums(preds, sems), FIX_A["input_checksums"])
    n = [int(FIX_A[f"a{i}_n"][0]) for i in range(4)]
    assert min(n[:3]) > 40_000 and int(FIX_A["a3_n_queries"][0]) < 100                    # the mean-IoU keep dropped queries
    assert n[3] < n[0], "the occupancy gate dropped rows"
    assert ((FIX_A["a3_pan"] != 0) & (FIX_A["a3_sem"] == 0)).any(), "a stuff class merged"
    assert len([k for k in FIX_A.files if k.startswith("a_match")]) == 2


def test_torch_confidence_outputs_match_reference_fixture_a():
    from pasco_b200 import ensemble as E
    preds, sems, Ts = GP.scene_a()
    thr = MANIFEST["a"]["thresholds"]
    sem_denses = E.ensemble_sem_compl(sems, Ts)
    out = E.ensemble_panop(preds, sem_denses, Ts, iou_threshold=thr["iou_threshold"])
    for i, (o, sd) in enumerate(zip(out, sem_denses)):
        prob, lin = o["voxel_probs"]
        order = torch.argsort(lin)
        pan, sem, conf, infos = E.panoptic_inference_with_confidence(prob[order], o["query_probs"][0],
                                                                     thr["overlap_threshold"], thr["object_mask_threshold"],
                                                                     GP.THING_IDS)
        flat = sd.reshape(sd.shape[0], -1)
        _check_fixture_a(i, lin[order], pan, sem, conf, infos, flat.argmax(0), flat.max(0)[0], prob.shape[1])


@pytest.mark.gpu
def test_postprocess_matches_reference_fixture_a():
    from pasco_b200 import predict as P
    thr = MANIFEST["a"]["thresholds"]
    preds, sems, Ts = _scene_a(torch.device("cuda"))
    matches = []
    got = P.postprocess(preds, sems, Ts, matches=matches, **thr)
    assert len(got) == 4 and len(matches) == 2
    for s, (ai, bi) in enumerate(matches):                               # the reference's Hungarian assignments
        assert np.array_equal(np.stack([ai, bi]), FIX_A[f"a_match{s}"]), s
    for i, e in enumerate(got):
        _check_fixture_a(i, e["lin"], e["panoptic_seg"], e["semantic_seg"], e["vox_confidence"], e["segments_info"],
                         P.to_dense(e, "ssc_pred"), P.to_dense(e, "ssc_confidence"), e["query_probs"].shape[0])


@pytest.mark.gpu
def test_pasconet_predict_matches_reference_fixture_b():
    """PascoNet.predict on the net_cfg1 scene at M = 2 (calibrated running statistics of net_cfg1_infer_m2.npz) against the
    reference's Net.forward(return_ensemble=True) + panoptic_inference, with the eval tests' near-tie tolerance: the
    forward agrees to rounding, so a few argmax near-ties may move rows; everything else must agree."""
    from pasco_b200 import ops, predict as P
    ops.set_precision("fp32")
    meta = parity.INFER_MANIFEST["cases"]["m2"]
    net, _ = parity.load_eval(parity.pasconet(2), "m2")
    b = parity.scene(meta, 2)
    got = net.predict(b["in_feats"], b["in_coords"], b["global_min_Cs"], b["global_max_Cs"], b["min_Cs"], b["max_Cs"],
                      GP.poses()[:2], **MANIFEST["b"]["thresholds"])
    z = FIX_B
    assert len(got) == 3
    rep = {}
    for i, e in enumerate(got):
        n_ref = int(z[f"b{i}_n"][0])
        n = e["lin"].numel()
        assert abs(n - n_ref) <= max(2, 0.002 * n_ref), (i, n, n_ref)
        assert len(e["segments_info"]) == len(z[f"b{i}_segments"])
        cats = sorted(s["category_id"] for s in e["segments_info"])
        assert cats == sorted(z[f"b{i}_segments"][:, 2].tolist())
        if n_ref:
            lin = e["lin"].cpu().numpy()
            ref_lin = z[f"b{i}_lin"]
            hit = np.isin(ref_lin, lin)
            pos = np.searchsorted(lin, ref_lin[hit])
            pan_ok = np.mean(e["panoptic_seg"].cpu().numpy()[pos] == z[f"b{i}_pan"][hit])
            sem_ok = np.mean(e["semantic_seg"].cpu().numpy()[pos] == z[f"b{i}_sem"][hit])
            conf = e["vox_confidence"].cpu().numpy()
            dconf = np.abs(conf[pos] - z[f"b{i}_conf"][hit])
            rep[i] = (float(hit.mean()), float(pan_ok), float(sem_ok), float(np.percentile(dconf, 99)))
            assert hit.mean() >= 0.995 and pan_ok >= 0.99 and sem_ok >= 0.99, rep[i]
            assert np.percentile(dconf, 99) <= 1e-3, rep[i]
        sc = P.to_dense(e, "ssc_confidence").reshape(-1).cpu()
        sp = P.to_dense(e, "ssc_pred").reshape(-1).cpu()
        ref = z[f"b{i}_ssc_sums"]
        assert abs(float(sc.double().sum()) - ref[0]) <= 1e-4 * ref[0], (i, float(sc.double().sum()), ref[0])
        assert abs(int((sp != 0).sum()) - int(ref[1])) <= max(2, 0.002 * ref[1])
        assert np.mean(sp[::GP.SUBSAMPLE].numpy() == z[f"b{i}_ssc_pred_sub"]) >= 0.995
    print("fixture (b): per entry (row hit rate, panoptic agreement, semantic agreement, p99 |Δconf|):", rep)
